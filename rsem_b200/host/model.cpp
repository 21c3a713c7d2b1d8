// Host-side model bookkeeping: the O(table) parts of the reference's four model classes
// (initial parameters, estimateFromReads, init/collect/finish, calcMW, read/write of .model).
// The O(hits x read length) parts (getConPrb, update) run on the GPU (csrc/model_kernels.cu).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "host.hpp"

namespace host {

// ---- LenDist ----------------------------------------------------------------------------------------
void LenDistH::reset(int minL, int maxL) {  // LenDist.h:17-32
    lb = minL - 1;
    ub = maxL;
    span = ub - lb;
    if (span <= 0) die("Length distribution has an empty support!");
    pdf.assign(span + 1, 0.0);
    cdf.assign(span + 1, 0.0);
    for (int i = 1; i <= span; ++i) {
        pdf[i] = 1.0 / span;
        cdf[i] = i * 1.0 / span;
    }
}
void LenDistH::zero() {
    std::fill(pdf.begin(), pdf.end(), 0.0);
    std::fill(cdf.begin(), cdf.end(), 0.0);
}
void LenDistH::finish() {  // LenDist.h:186-200
    double sum = 0.0;
    for (int i = 1; i <= span; ++i) sum += pdf[i];
    if (sum <= kEps) die("No valid read to estimate the length distribution!");
    for (int i = 1; i <= span; ++i) {
        pdf[i] = pdf[i] / sum;
        cdf[i] = cdf[i - 1] + pdf[i];
    }
    trim();
}
void LenDistH::trim() {  // LenDist.h:265-294: drop zero tails, which moves lb / ub
    int newlb, newub;
    for (newlb = 1; newlb <= span && pdf[newlb] < kEps; ++newlb) {}
    --newlb;
    for (newub = span; newub > newlb && pdf[newub] < kEps; --newub) {}
    if (newlb >= newub) die("Length distribution is empty after trimming!");
    if (newlb == 0 && newub == span) return;
    const int nspan = newub - newlb;
    std::vector<double> np(nspan + 1, 0.0), nc(nspan + 1, 0.0);
    for (int i = 1; i <= nspan; ++i) {
        np[i] = pdf[i + newlb];
        nc[i] = cdf[i + newlb];
    }
    pdf.swap(np);
    cdf.swap(nc);
    span = nspan;
    lb += newlb;
    ub = lb + span;
}
static double normal_cdf(double x, double mean, double sd) {  // boost::math::cdf(normal) == erfc form
    return 0.5 * erfc(-(x - mean) / (sd * sqrt(2.0)));
}
void LenDistH::set_as_normal(double mean, double sd, int minL, int maxL) {  // LenDist.h:91-179
    const int meanL = int(mean + .5);
    if (sd < kEps) {
        if (meanL < minL || meanL > maxL) {
            die("Length distribution's probability mass is not within the possible range! MeanL = " + std::to_string(meanL) +
                ", MinL = " + std::to_string(minL) + ", MaxL = " + std::to_string(maxL));
        }
        span = 1;
        lb = meanL - 1;
        ub = meanL;
        pdf.assign(2, 0.0);
        cdf.assign(2, 0.0);
        pdf[1] = cdf[1] = 1.0;
        return;
    }
    if (maxL - minL + 1 > kRange) {
        if (meanL <= minL) maxL = minL + kRange - 1;
        else if (meanL >= maxL) minL = maxL - kRange + 1;
        else {
            const double lg = mean - (minL - 0.5), rg = (maxL + 0.5) - mean, half = kRange / 2.0;
            if (lg < half) maxL = minL + kRange - 1;
            else if (rg < half) minL = maxL - kRange + 1;
            else { minL = int(mean - half + 1.0); maxL = int(mean + half); }
        }
    }
    lb = minL - 1;
    ub = maxL;
    span = ub - lb;
    pdf.assign(span + 1, 0.0);
    cdf.assign(span + 1, 0.0);
    double sum = 0.0, old_val = normal_cdf(minL - 0.5, mean, sd);
    for (int i = 1; i <= span; ++i) {
        const double val = normal_cdf(lb + i + 0.5, mean, sd);
        pdf[i] = val - old_val;
        sum += pdf[i];
        old_val = val;
    }
    for (int i = 1; i <= span; ++i) {
        pdf[i] /= sum;
        cdf[i] = cdf[i - 1] + pdf[i];
    }
    trim();
}
double LenDistH::adj(int len, int refL) const {
    if (len <= lb || len > ub || refL <= lb) return 0.0;
    return pdf[len - lb] / cdf[std::min(ub, refL) - lb];
}
double LenDistH::adj_cum(int len, int refL) const { return cdf[len - lb] / cdf[std::min(ub, refL) - lb]; }
void LenDistH::write(FILE* fo) const {
    fprintf(fo, "%d %d %d\n", lb, ub, span);
    for (int i = 1; i < span; ++i) fprintf(fo, "%.10g ", pdf[i]);
    fprintf(fo, "%.10g\n", pdf[span]);
}
void LenDistH::read(FILE* fi) {
    if (fscanf(fi, "%d %d %d", &lb, &ub, &span) != 3) die("Cannot parse a length distribution in the .model file!");
    pdf.assign(span + 1, 0.0);
    cdf.assign(span + 1, 0.0);
    for (int i = 1; i <= span; ++i) {
        if (fscanf(fi, "%lf", &pdf[i]) != 1) die("Cannot parse a length distribution in the .model file!");
        cdf[i] = cdf[i - 1] + pdf[i];
    }
    trim();
}

// ---- initial tables ---------------------------------------------------------------------------------
static void init_profile(std::vector<double>& p, int rows) {  // Profile.h:47-72
    p.assign((size_t)rows * 25, 0.0);
    const double probN = 1e-5, portionC = 0.99;
    for (int i = 0; i < rows; ++i) {
        double* q = &p[(size_t)i * 25];
        for (int j = 0; j < 4; ++j) {
            q[j * 5 + 4] = probN;
            const double probC = portionC * (1.0 - probN);
            const double probO = (1.0 - portionC) / 3 * (1.0 - probN);
            for (int k = 0; k < 4; ++k) q[j * 5 + k] = (j == k ? probC : probO);
        }
        q[4 * 5 + 4] = probN;
        for (int k = 0; k < 4; ++k) q[4 * 5 + k] = (1.0 - probN) / 4;
    }
}
static void init_qprofile(std::vector<double>& p) {  // QProfile.h:45-76
    p.assign(2500, 0.0);
    const double probN = 1e-5;
    for (int i = 0; i < 100; ++i) {
        double* q = &p[(size_t)i * 25];
        for (int j = 0; j < 4; ++j) {
            q[j * 5 + 4] = probN;
            double probO = exp(-i / 10.0 * log(10.0));
            double probC = 1.0 - probO;
            probO /= 3;
            probC *= (1.0 - probN);
            probO *= (1.0 - probN);
            for (int k = 0; k < 4; ++k) q[j * 5 + k] = (j == k ? probC : probO);
        }
        q[4 * 5 + 4] = probN;
        for (int k = 0; k < 4; ++k) q[4 * 5 + k] = (1.0 - probN) / 4;
    }
}
static void init_rspd(std::vector<double>& pdf, std::vector<double>& cdf, int B) {  // RSPD.h:21-33
    pdf.assign(B + 2, 0.0);
    cdf.assign(B + 2, 0.0);
    for (int i = 1; i <= B; ++i) {
        pdf[i] = 1.0 / B;
        cdf[i] = i * 1.0 / B;
    }
}

void HostModel::init_master(int model_type, const ModelParamsH& p, const RefData* r) {
    type = model_type;
    mp = p;
    refs = r;
    ori[0] = p.probF;
    ori[1] = 1.0 - p.probF;
    gld.reset(p.minL, p.maxL);
    has_mld = false;
    if (paired()) {  // PairedEndQModel.h:66-74
        mld.reset(p.mate_minL, p.mate_maxL);
        has_mld = true;
    } else if (p.mean >= kEps) {  // SingleQModel.h:69-72
        mld.reset(p.mate_minL, p.mate_maxL);
        has_mld = true;
    }
    init_rspd(rspd_pdf, rspd_cdf, p.estRSPD ? p.B : 20);  // RSPD(estRSPD) default B = 20 (RSPD.h:13)
    if (hasq()) {
        qd_init.assign(100, 0.0);
        qd_tran.assign(100 * 100, 0.0);
        pro_len = 0;
        init_qprofile(profile);
    } else {
        pro_len = p.maxL;  // Profile(params.maxL), SingleModel.h:76
        init_profile(profile, pro_len);
    }
    noise_p.assign(n_noise(), 0.0);
    noise_c.assign(n_noise(), 0.0);
    mw.assign((size_t)p.M + 1, 0.0);
}

// ---- estimateFromReads (SingleQModel.h:283-327, PairedEndQModel.h:241-290) -----------------------------
// One pass over the un / alignable / max read sets: read (mate) length histogram, QualDist counts, base counts of the
// unalignable reads.  All of them are integer counts, so per-thread partial sums merge exactly.
namespace {
struct ReadCounts {
    std::vector<double> len, qd_init, qd_tran, noise_c;
    bool bad_len = false;
};
}  // namespace

void HostModel::estimate_from_reads(const std::string& imd, ReadStore& alignable, Sidecar* sc) {
    LenDistH& d = (paired() || has_mld) ? mld : gld;
    d.zero();
    int n_warns = 0;
    for (int tag = 0; tag < 3; ++tag) {
        if (mp.N[tag] == 0) continue;
        ReadStore local;
        ReadStore& rs = tag == 1 ? alignable : local;
        std::vector<std::string> short_names;
        uint64_t n_short = 0;
        const int n_warns_before = n_warns;
        if (sc) {  // already decoded by bin/rsem-parse-alignments (binary side-car): only the lowq flags are derived here
            rs = std::move(sc->reads[tag]);
            finish_sidecar_reads(rs, sc->shorts[tag], refs->has_polyA, mp.seedLen, &short_names, &n_short);
        } else {
            parse_reads(imd, tag, type, refs->has_polyA, mp.seedLen, rs, &short_names, &n_short);
        }
        const int T = std::max(1, std::min<int>(g_io_threads, (int)(rs.n / 8192) + 1));
        std::vector<ReadCounts> part(T);
        parallel_ranges((size_t)rs.n, T, [&](size_t b, size_t e, int t) {
            ReadCounts& pc = part[t];
            pc.len.assign(d.span + 1, 0.0);
            if (hasq()) { pc.qd_init.assign(100, 0.0); pc.qd_tran.assign(100 * 100, 0.0); }
            if (tag == 0) pc.noise_c.assign(n_noise(), 0.0);
            for (size_t i = b; i < e; ++i) {
                if (rs.lowq[i]) continue;
                for (int k = 0; k < rs.n_mates; ++k) {
                    const uint64_t o = rs.off[k][i];
                    const int len = (int)(rs.off[k][i + 1] - o);
                    if (!(len > d.lb && len <= d.ub)) { pc.bad_len = true; continue; }  // LenDist.h:47 assert
                    pc.len[len - d.lb] += 1.0;
                    const uint8_t* bq = rs.base[k].data() + o;
                    if (hasq()) {  // QualDist::update, QualDist.h:54-63
                        const uint8_t* q = rs.qual[k].data() + o;
                        pc.qd_init[q[0]] += 1.0;
                        for (int j = 1; j < len; ++j) pc.qd_tran[(size_t)q[j - 1] * 100 + q[j]] += 1.0;
                        if (tag == 0) for (int j = 0; j < len; ++j) pc.noise_c[(size_t)q[j] * 5 + bq[j]] += 1.0;  // updateC
                    } else if (tag == 0) {
                        for (int j = 0; j < len; ++j) pc.noise_c[bq[j]] += 1.0;
                    }
                }
            }
        });
        for (const ReadCounts& pc : part) {
            if (pc.bad_len) die("A read has a length outside the allowed range!");
            for (size_t j = 0; j < pc.len.size(); ++j) d.pdf[j] += pc.len[j];
            for (size_t j = 0; j < pc.qd_init.size(); ++j) qd_init[j] += pc.qd_init[j];
            for (size_t j = 0; j < pc.qd_tran.size(); ++j) qd_tran[j] += pc.qd_tran[j];
            for (size_t j = 0; j < pc.noise_c.size(); ++j) noise_c[j] += pc.noise_c[j];
        }
        // The reference prints the first 50 warnings; PairedEndQModel.h:272 never increments n_warns (reference
        // quirk), so that model warns about every short pair and prints no total.
        for (const std::string& name : short_names) {
            if (type != 3 && ++n_warns > 50) break;
            if (!paired())
                fprintf(stderr, "Warning: Read %s is ignored due to read length < seed length (= %d)!\n", name.c_str(), mp.seedLen);
            else
                fprintf(stderr, "Warning: Read %s is ignored due to at least one of the mates' length < seed length (= %d)!\n", name.c_str(), mp.seedLen);
        }
        if (type != 3) n_warns = (int)std::min<uint64_t>((uint64_t)n_warns_before + n_short, 1u << 30);
        if (g_verbose) printf("estimateFromReads, N%d finished.\n", tag);
    }
    if (n_warns > 0) fprintf(stderr, "Warning: There are %d reads ignored in total.\n", n_warns);
    d.finish();
    if (!paired() && mp.mean >= kEps) {  // SingleQModel.h:318-321
        gld.set_as_normal(mp.mean, mp.sd, std::max(mld.minL(), gld.minL()), gld.maxL());
    }
    if (hasq()) {  // QualDist::finish, QualDist.h:65-79
        double sum = 0.0;
        for (int i = 0; i < 100; ++i) sum += qd_init[i];
        for (int i = 0; i < 100; ++i) qd_init[i] /= sum;
        for (int i = 0; i < 100; ++i) {
            sum = 0.0;
            for (int j = 0; j < 100; ++j) sum += qd_tran[(size_t)i * 100 + j];
            if (sum <= 0.0) continue;
            for (int j = 0; j < 100; ++j) qd_tran[(size_t)i * 100 + j] /= sum;
        }
    }
    // Noise(Q)Profile::calcInitParams: pseudo count 1 (NoiseQProfile.h:99-111, NoiseProfile.h:91-101)
    if (hasq()) {
        for (int i = 0; i < 100; ++i) {
            double sum = 0.0;
            for (int j = 0; j < 5; ++j) sum += 1.0 + noise_c[i * 5 + j];
            for (int j = 0; j < 5; ++j) noise_p[i * 5 + j] = (noise_c[i * 5 + j] + 1.0) / sum;
        }
    } else {
        double sum = 0.0;
        for (int j = 0; j < 5; ++j) sum += 1.0 + noise_c[j];
        for (int j = 0; j < 5; ++j) noise_p[j] = (1.0 + noise_c[j]) / sum;
    }
    calc_mw();
}

// ---- init(); collect(helpers); finish() -----------------------------------------------------------------
void HostModel::rebuild(const rsem_b200_model_stats& st) {
    if (paired()) {  // gld re-estimated from insert-length posteriors on the ORIGINAL support (PairedEndQModel.h:72,168,292-306)
        gld.lb = st.gld_lb;
        gld.span = st.gld_span;
        gld.ub = gld.lb + gld.span;
        gld.pdf.assign(st.gld_pdf, st.gld_pdf + gld.span + 1);
        gld.pdf[0] = 0.0;
        gld.cdf.assign(gld.span + 1, 0.0);
        gld.finish();
    }
    if (mp.estRSPD) {  // RSPD::finish, RSPD.h:116-129
        const int B = mp.B;
        double sum = 0.0;
        for (int i = 1; i <= B; ++i) { rspd_pdf[i] = st.rspd_pdf[i]; sum += rspd_pdf[i]; }
        rspd_cdf[0] = 0.0;
        for (int i = 1; i <= B; ++i) {
            rspd_pdf[i] /= sum;
            rspd_cdf[i] = rspd_cdf[i - 1] + rspd_pdf[i];
        }
    }
    {   // (Q)Profile::finish, Profile.h:98-112 / QProfile.h:95-109
        const size_t rows = hasq() ? 100 : (size_t)pro_len;
        for (size_t i = 0; i < rows; ++i)
            for (int j = 0; j < 5; ++j) {
                const double* src = st.profile + (i * 5 + j) * 5;
                double* dst = &profile[(i * 5 + j) * 5];
                double sum = 0.0;
                for (int k = 0; k < 5; ++k) sum += src[k];
                if (sum < kEps) { for (int k = 0; k < 5; ++k) dst[k] = 0.0; continue; }
                for (int k = 0; k < 5; ++k) dst[k] = src[k] / sum;
            }
    }
    if (hasq()) {  // NoiseQProfile::finish, NoiseQProfile.h:81-96
        for (int i = 0; i < 100; ++i) {
            double sum = 0.0;
            for (int j = 0; j < 5; ++j) sum += st.noise_profile[i * 5 + j] + noise_c[i * 5 + j];
            if (sum <= 0.0) { for (int j = 0; j < 5; ++j) noise_p[i * 5 + j] = st.noise_profile[i * 5 + j]; continue; }
            for (int j = 0; j < 5; ++j) noise_p[i * 5 + j] = (st.noise_profile[i * 5 + j] + noise_c[i * 5 + j]) / sum;
        }
    } else {  // NoiseProfile::finish, NoiseProfile.h:78-89
        double sum = 0.0;
        for (int j = 0; j < 5; ++j) sum += st.noise_profile[j] + noise_c[j];
        if (sum <= kEps) { for (int j = 0; j < 5; ++j) noise_p[j] = st.noise_profile[j]; }
        else for (int j = 0; j < 5; ++j) noise_p[j] = (st.noise_profile[j] + noise_c[j]) / sum;
    }
    // Single models recompute mw only when RSPD is estimated; paired models always (SingleQModel.h:335-341, PairedEndQModel.h:299-306)
    if (paired() || mp.estRSPD) calc_mw();
}

double HostModel::rspd_eval_cdf(int fpos, int fullLen) const {  // RSPD.h:63-68
    const int B = mp.estRSPD ? mp.B : 20;
    const int i = (int)(((long long)fpos) * B / fullLen);
    const double val = fpos * 1.0 / fullLen * B;
    return rspd_cdf[i] + (val - i) * rspd_pdf[i + 1];
}
double HostModel::rspd_adj(int fpos, int effL, int fullLen) const {  // RSPD.h:70-75
    if (!mp.estRSPD) return 1.0 / effL;
    const double denom = rspd_eval_cdf(effL, fullLen);
    return denom >= kEps ? (rspd_eval_cdf(fpos + 1, fullLen) - rspd_eval_cdf(fpos, fullLen)) / denom : 0.0;
}

// ---- calcMW (SingleQModel.h:482-544, PairedEndQModel.h:445-479) -------------------------------------------
void HostModel::calc_mw() {
    const int M = mp.M, seedLen = mp.seedLen;
    std::fill(mw.begin(), mw.end(), 0.0);
    mw[0] = 1.0;
    if (!refs->has_polyA) {  // no mask bit is ever set without poly(A) tails (RefSeq.h:31-37): value stays 0
        // single-end models still add the "reverse strand" term over seedPos in [end, totLen - seedLen], which is
        // empty when totLen == fullLen and fullLen >= seedLen ... but not when fullLen < seedLen; fall through then.
        bool trivial = true;
        if (!paired())
            for (int i = 1; i <= M && trivial; ++i) trivial = refs->full_len[i] >= seedLen;
        if (trivial) { for (int i = 1; i <= M; ++i) mw[i] = 1.0; return; }
    }
    const double probF = ori[0], probR = ori[1];
    for (int i = 1; i <= M; ++i) {
        const int totLen = refs->tot_len[i], fullLen = refs->full_len[i];
        double value = 0.0;
        if (paired()) {
            const int end = std::min(fullLen, totLen - gld.minL() + 1);
            for (int seedPos = 0; seedPos < end; ++seedPos)
                if (refs->mask(i, seedPos)) {
                    const int minL = gld.minL(), maxL = std::min(gld.maxL(), totLen - seedPos);
                    for (int fragLen = minL; fragLen <= maxL; ++fragLen) {
                        const int effL = std::min(fullLen, totLen - fragLen + 1);
                        value += gld.adj(fragLen, totLen) * rspd_adj(seedPos, effL, fullLen);
                    }
                }
        } else {
            const int end = std::min(fullLen, totLen - seedLen + 1);
            for (int seedPos = 0; seedPos < end; ++seedPos)
                if (refs->mask(i, seedPos)) {
                    int minL = gld.minL(), maxL = std::min(gld.maxL(), totLen - seedPos);
                    for (int fragLen = minL; fragLen <= maxL; ++fragLen) {  // forward
                        const int effL = std::min(fullLen, totLen - fragLen + 1);
                        const double factor = has_mld ? mld.adj_cum(std::min(mld.maxL(), fragLen), fragLen) : 1.0;
                        value += probF * gld.adj(fragLen, totLen) * rspd_adj(seedPos, effL, fullLen) * factor;
                    }
                    maxL = std::min(gld.maxL(), seedPos + seedLen);
                    for (int fragLen = minL; fragLen <= maxL; ++fragLen) {  // reverse
                        const int pfpos = seedPos - (fragLen - seedLen);
                        const int effL = std::min(fullLen, totLen - fragLen + 1);
                        const double factor = has_mld ? mld.adj_cum(std::min(mld.maxL(), fragLen), fragLen) : 1.0;
                        value += probR * gld.adj(fragLen, totLen) * rspd_adj(pfpos, effL, fullLen) * factor;
                    }
                }
            for (int seedPos = end; seedPos <= totLen - seedLen; ++seedPos) {  // reverse-strand masking
                const int minL = std::max(gld.minL(), seedPos + seedLen - fullLen + 1);
                const int maxL = std::min(gld.maxL(), seedPos + seedLen);
                for (int fragLen = minL; fragLen <= maxL; ++fragLen) {
                    const int pfpos = seedPos - (fragLen - seedLen);
                    const int effL = std::min(fullLen, totLen - fragLen + 1);
                    const double factor = has_mld ? mld.adj_cum(std::min(mld.maxL(), fragLen), fragLen) : 1.0;
                    value += probR * gld.adj(fragLen, totLen) * rspd_adj(pfpos, effL, fullLen) * factor;
                }
            }
        }
        mw[i] = 1.0 - value;
        if (mw[i] < 1e-8) mw[i] = 0.0;
    }
}

void HostModel::fill_abi(rsem_b200_model& m) const {
    memset(&m, 0, sizeof m);
    m.model_type = type;
    m.M = mp.M;
    m.seed_len = mp.seedLen;
    m.est_rspd = mp.estRSPD;
    m.rspd_B = mp.estRSPD ? mp.B : 20;
    m.has_mld = has_mld;
    m.pro_len = pro_len;
    m.ori[0] = ori[0];
    m.ori[1] = ori[1];
    m.gld = rsem_b200_lendist{gld.lb, gld.ub, gld.span, gld.pdf.data(), gld.cdf.data()};
    if (has_mld) m.mld = rsem_b200_lendist{mld.lb, mld.ub, mld.span, mld.pdf.data(), mld.cdf.data()};
    m.rspd_pdf = rspd_pdf.data();
    m.rspd_cdf = rspd_cdf.data();
    m.profile = profile.data();
    m.noise_profile = noise_p.data();
    m.mw = mw.data();
}

// ---- .model (model_file_description.txt; SingleQModel.h:383-411, PairedEndQModel.h:346-369) -------------------
static void write_profile(FILE* fo, const std::vector<double>& p, int rows) {
    fprintf(fo, "%d %d\n", rows, 5);
    for (int i = 0; i < rows; ++i) {
        for (int j = 0; j < 5; ++j) {
            for (int k = 0; k < 4; ++k) fprintf(fo, "%.10g ", p[((size_t)i * 5 + j) * 5 + k]);
            fprintf(fo, "%.10g\n", p[((size_t)i * 5 + j) * 5 + 4]);
        }
        if (i < rows - 1) fprintf(fo, "\n");
    }
}

void HostModel::write(const std::string& path) const {
    FILE* fo = fopen(path.c_str(), "w");
    if (!fo) die("Cannot open " + path + " for writing!");
    fprintf(fo, "%d\n\n", type);
    fprintf(fo, "%.10g\n\n", ori[0]);
    gld.write(fo);
    fprintf(fo, "\n");
    if (paired()) { mld.write(fo); fprintf(fo, "\n"); }
    else {
        if (has_mld) { fprintf(fo, "1\n"); mld.write(fo); } else fprintf(fo, "0\n");
        fprintf(fo, "\n");
    }
    fprintf(fo, "%d\n", mp.estRSPD ? 1 : 0);  // RSPD::write, RSPD.h:175-184
    if (mp.estRSPD) {
        fprintf(fo, "%d\n", mp.B);
        for (int i = 1; i < mp.B; ++i) fprintf(fo, "%.10g ", rspd_pdf[i]);
        fprintf(fo, "%.10g\n", rspd_pdf[mp.B]);
    }
    fprintf(fo, "\n");
    if (hasq()) {  // QualDist::write, QualDist.h:103-112
        fprintf(fo, "%d\n", 100);
        for (int i = 0; i < 99; ++i) fprintf(fo, "%.10g ", qd_init[i]);
        fprintf(fo, "%.10g\n", qd_init[99]);
        for (int i = 0; i < 100; ++i) {
            for (int j = 0; j < 99; ++j) fprintf(fo, "%.10g ", qd_tran[(size_t)i * 100 + j]);
            fprintf(fo, "%.10g\n", qd_tran[(size_t)i * 100 + 99]);
        }
        fprintf(fo, "\n");
    }
    write_profile(fo, profile, hasq() ? 100 : pro_len);
    fprintf(fo, "\n");
    if (hasq()) {  // NoiseQProfile::write
        fprintf(fo, "%d %d\n", 100, 5);
        for (int i = 0; i < 100; ++i) {
            for (int j = 0; j < 4; ++j) fprintf(fo, "%.10g ", noise_p[i * 5 + j]);
            fprintf(fo, "%.10g\n", noise_p[i * 5 + 4]);
        }
    } else {  // NoiseProfile::write
        fprintf(fo, "%d\n", 5);
        for (int j = 0; j < 4; ++j) fprintf(fo, "%.10g ", noise_p[j]);
        fprintf(fo, "%.10g\n", noise_p[4]);
    }
    fprintf(fo, "\n%d\n", mp.M);
    for (int i = 0; i < mp.M; ++i) fprintf(fo, "%.15g ", mw[i]);
    fprintf(fo, "%.15g\n", mw[mp.M]);
    fclose(fo);
}

void HostModel::read_for_gibbs(const std::string& path, int M, int& model_type, LenDistH& gld, std::vector<double>& mw) {
    FILE* fi = fopen(path.c_str(), "r");
    if (!fi) die("Cannot open " + path + "! It may not exist.");
    auto need = [&](bool ok) { if (!ok) die("Cannot parse " + path + "!"); };
    double d;
    int v;
    need(fscanf(fi, "%d", &model_type) == 1);
    need(model_type >= 0 && model_type <= 3);
    need(fscanf(fi, "%lf", &d) == 1);  // Orientation
    gld.read(fi);
    LenDistH mld;
    if (model_type >= 2) mld.read(fi);
    else {
        need(fscanf(fi, "%d", &v) == 1);
        if (v > 0) mld.read(fi);
    }
    need(fscanf(fi, "%d", &v) == 1);  // RSPD
    if (v != 0) {
        int B;
        need(fscanf(fi, "%d", &B) == 1);
        for (int i = 0; i < B; ++i) need(fscanf(fi, "%lf", &d) == 1);
    }
    if (model_type & 1) {  // QualDist
        need(fscanf(fi, "%d", &v) == 1 && v == 100);
        for (int i = 0; i < 100 + 100 * 100; ++i) need(fscanf(fi, "%lf", &d) == 1);
    }
    int rows, ncodes;  // (Q)Profile
    need(fscanf(fi, "%d %d", &rows, &ncodes) == 2 && ncodes == 5);
    for (int i = 0; i < rows * 25; ++i) need(fscanf(fi, "%lf", &d) == 1);
    if (model_type & 1) {  // NoiseQProfile
        need(fscanf(fi, "%d %d", &rows, &ncodes) == 2);
        for (int i = 0; i < rows * ncodes; ++i) need(fscanf(fi, "%lf", &d) == 1);
    } else {
        need(fscanf(fi, "%d", &ncodes) == 1);
        for (int i = 0; i < ncodes; ++i) need(fscanf(fi, "%lf", &d) == 1);
    }
    mw.clear();
    if (fscanf(fi, "%d", &v) == 1 && v == M) {
        mw.resize((size_t)M + 1);
        for (int i = 0; i <= M; ++i) need(fscanf(fi, "%lf", &mw[i]) == 1);
    }
    fclose(fi);
    if (mw.empty()) die("The .model file does not carry mask weights for this reference!");
}

// Model::read (SingleModel.h:356-381, SingleQModel.h:383-411, PairedEndModel.h:296-317, PairedEndQModel.h:316-343)
void HostModel::read(const std::string& path, int M, int* file_M) {
    FILE* fi = fopen(path.c_str(), "r");
    if (!fi) die("Cannot open " + path + "! It may not exist.");
    auto need = [&](bool ok) { if (!ok) die("Cannot parse " + path + "!"); };
    int v;
    need(fscanf(fi, "%d", &type) == 1 && type >= 0 && type <= 3);
    need(fscanf(fi, "%lf", &ori[0]) == 1);  // Orientation.h:26-29
    ori[1] = 1.0 - ori[0];
    gld.read(fi);
    if (paired()) { mld.read(fi); has_mld = true; }
    else {
        need(fscanf(fi, "%d", &v) == 1);
        has_mld = v > 0;
        if (has_mld) mld.read(fi);
    }
    need(fscanf(fi, "%d", &v) == 1);  // RSPD.h:138-167
    mp.estRSPD = v != 0;
    if (mp.estRSPD) need(fscanf(fi, "%d", &mp.B) == 1 && mp.B >= 1);
    const int B = mp.estRSPD ? mp.B : 20;
    rspd_pdf.assign(B + 2, 0.0);
    rspd_cdf.assign(B + 2, 0.0);
    for (int i = 1; i <= B; ++i) {
        if (mp.estRSPD) need(fscanf(fi, "%lf", &rspd_pdf[i]) == 1);
        else rspd_pdf[i] = 1.0 / B;
        rspd_cdf[i] = mp.estRSPD ? rspd_cdf[i - 1] + rspd_pdf[i] : i * 1.0 / B;
    }
    if (hasq()) {  // QualDist.h:94-104
        need(fscanf(fi, "%d", &v) == 1 && v == 100);
        qd_init.assign(100, 0.0);
        qd_tran.assign(100 * 100, 0.0);
        for (double& d : qd_init) need(fscanf(fi, "%lf", &d) == 1);
        for (double& d : qd_tran) need(fscanf(fi, "%lf", &d) == 1);
    }
    int rows, ncodes;  // QProfile.h:129-137, Profile.h:133-149
    need(fscanf(fi, "%d %d", &rows, &ncodes) == 2 && ncodes == 5 && rows >= 0 && (!hasq() || rows == 100));
    pro_len = hasq() ? 0 : rows;
    profile.assign((size_t)rows * 25, 0.0);
    for (double& d : profile) need(fscanf(fi, "%lf", &d) == 1);
    if (hasq()) {  // NoiseQProfile.h:132-143
        need(fscanf(fi, "%d %d", &rows, &ncodes) == 2 && rows == 100 && ncodes == 5);
        noise_p.assign(500, 0.0);
    } else {  // NoiseProfile.h:119-127
        need(fscanf(fi, "%d", &ncodes) == 1 && ncodes == 5);
        noise_p.assign(5, 0.0);
    }
    for (double& d : noise_p) need(fscanf(fi, "%lf", &d) == 1);
    mw.clear();
    const bool has_M = fscanf(fi, "%d", &v) == 1;
    if (file_M) *file_M = has_M ? v : 0;
    if (has_M && v == M) {
        mw.resize((size_t)M + 1);
        for (int i = 0; i <= M; ++i) need(fscanf(fi, "%lf", &mw[i]) == 1);
    }
    mp.M = M;
    fclose(fi);
}

// ---- WriteResults.h:24-104 ---------------------------------------------------------------------------------
void calc_eel(const RefData& refs, const LenDistH& gld, std::vector<double>& eel) {
    const int lb = gld.lb, ub = gld.ub, span = gld.span;
    std::vector<double> clen(span + 1, 0.0);
    for (int i = 1; i <= span; ++i) clen[i] = clen[i - 1] + gld.pdf[i] * (lb + i);
    eel.assign((size_t)refs.M + 1, 0.0);
    for (int i = 1; i <= refs.M; ++i) {
        const int totLen = refs.tot_len[i], fullLen = refs.full_len[i];
        const int pos1 = std::max(std::min(totLen - fullLen + 1, ub) - lb, 0);
        const int pos2 = std::max(std::min(totLen, ub) - lb, 0);
        if (pos2 == 0) { eel[i] = 0.0; continue; }
        eel[i] = fullLen * gld.cdf[pos1] + ((gld.cdf[pos2] - gld.cdf[pos1]) * (totLen + 1) - (clen[pos2] - clen[pos1]));
        if (eel[i] < kMinEel) eel[i] = 0.0;
    }
}

void polish_theta(std::vector<double>& theta, const std::vector<double>& eel, const std::vector<double>& mw) {
    const int M = (int)theta.size() - 1;
    double sum = 0.0;
    for (int i = 0; i <= M; ++i) {
        if (i > 0 && (mw[i] < kEps || eel[i] < kEps)) { theta[i] = 0.0; continue; }
        theta[i] = theta[i] / mw[i];
        sum += theta[i];
    }
    if (!(sum >= kEps)) die("No effective length is no less than1 !");
    for (int i = 0; i <= M; ++i) theta[i] /= sum;
}

void expression_values(const std::vector<double>& theta, const std::vector<double>& eel, std::vector<double>& tpm,
                       std::vector<double>& fpkm) {
    const int M = (int)theta.size() - 1;
    std::vector<double> frac(M + 1, 0.0);
    double denom = 0.0;
    for (int i = 1; i <= M; ++i)
        if (eel[i] >= kEps) { frac[i] = theta[i]; denom += frac[i]; }
    if (denom < kEps) denom = 1.0;
    for (int i = 1; i <= M; ++i) frac[i] /= denom;
    fpkm.assign(M + 1, 0.0);
    for (int i = 1; i <= M; ++i)
        if (eel[i] >= kEps) fpkm[i] = frac[i] * 1e9 / eel[i];
    tpm.assign(M + 1, 0.0);
    denom = 0.0;
    for (int i = 1; i <= M; ++i) denom += fpkm[i];
    if (denom < kEps) denom = 1.0;
    for (int i = 1; i <= M; ++i) tpm[i] = fpkm[i] / denom * 1e6;
}

}  // namespace host
