/*
 * rsem_oracle.c - TEST INFRASTRUCTURE ONLY (see rsem_oracle.h for the rules).
 * Sequential restatement of the reference algorithms; loops keep the reference's order of
 * floating-point operations wherever the reference's order is defined.
 */
#include "rsem_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define RO_EPS 1e-300 /* utils.h:18 EPSILON */

/* ------------------------------------------------------------------------------------------ */
/* E-step for one read range, EM.cpp:199-244                                                   */
static void estep_range(uint64_t lo, uint64_t hi, const uint64_t* row_ptr, const int32_t* sid,
                        const double* conprb, const double* ncpv, const double* theta, double* counts, double* post,
                        double* post0) {
    for (uint64_t i = lo; i < hi; ++i) {
        const uint64_t fr = row_ptr[i], to = row_ptr[i + 1];
        double f0 = theta[0] * ncpv[i]; /* EM.cpp:211-212 */
        if (f0 < RO_EPS) f0 = 0.0;
        double sum = f0;
        for (uint64_t j = fr; j < to; ++j) { /* EM.cpp:214-221 */
            double f = theta[abs(sid[j])] * conprb[j];
            if (f < RO_EPS) f = 0.0;
            sum += f;
        }
        if (sum >= RO_EPS) { /* EM.cpp:223-236 */
            f0 /= sum;
            counts[0] += f0;
            if (post0) post0[i] = f0;
            for (uint64_t j = fr; j < to; ++j) {
                const int t = abs(sid[j]);
                double f = theta[t] * conprb[j];
                if (f < RO_EPS) f = 0.0;
                f /= sum;
                counts[t] += f;
                if (post) post[j] = f;
            }
        } else if (post) { /* EM.cpp:237-243 */
            if (post0) post0[i] = 0.0;
            for (uint64_t j = fr; j < to; ++j) post[j] = 0.0;
        }
    }
}

void ro_estep(uint64_t N, const uint64_t* row_ptr, const int32_t* sid, const double* conprb, const double* ncpv,
              const double* theta, int32_t M, double* counts, double* post, double* post0, int32_t n_threads) {
    memset(counts, 0, sizeof(double) * ((size_t)M + 1));
    if (n_threads <= 1) {
        estep_range(0, N, row_ptr, sid, conprb, ncpv, theta, counts, post, post0);
        return;
    }
#ifdef _OPENMP
    /* contiguous read ranges with ~equal hit counts (EM.cpp:135-157), private count vectors,
     * serial merge (EM.cpp:385-389) */
    /* private count vectors are kept between calls (the reference allocates countvs[] once, EM.cpp:166-170) and
     * zeroed by their owning thread (first touch places them on that thread's NUMA node) */
    static double* priv = NULL;
    static size_t priv_cap = 0;
    const size_t need = (size_t)n_threads * ((size_t)M + 1);
    if (priv_cap < need) {
        free(priv);
        priv = (double*)malloc(need * sizeof(double));
        priv_cap = need;
    }
    const uint64_t H = row_ptr[N];
#pragma omp parallel num_threads(n_threads)
    {
        const int t = omp_get_thread_num(), T = omp_get_num_threads();
        memset(priv + (size_t)t * ((size_t)M + 1), 0, sizeof(double) * ((size_t)M + 1));
        uint64_t lo, hi;
        { /* first row whose start >= t * H / T */
            uint64_t target = (uint64_t)((__uint128_t)H * t / T), a = 0, b = N;
            while (a < b) { uint64_t mid = (a + b) >> 1; if (row_ptr[mid] < target) a = mid + 1; else b = mid; }
            lo = t == 0 ? 0 : a;
            target = (uint64_t)((__uint128_t)H * (t + 1) / T); a = 0; b = N;
            while (a < b) { uint64_t mid = (a + b) >> 1; if (row_ptr[mid] < target) a = mid + 1; else b = mid; }
            hi = t == T - 1 ? N : a;
        }
        estep_range(lo, hi, row_ptr, sid, conprb, ncpv, theta, priv + (size_t)t * ((size_t)M + 1), post, post0);
    }
    /* the reference merges serially (EM.cpp:385-389); the port splits the merge over transcripts so that a
     * bounded benchmark sample with many threads is not dominated by it */
#pragma omp parallel for num_threads(n_threads) schedule(static)
    for (int32_t k = 0; k <= M; ++k) {
        double acc = 0.0;
        for (int t = 0; t < n_threads; ++t) acc += priv[(size_t)t * ((size_t)M + 1) + k];
        counts[k] = acc;
    }
#else
    estep_range(0, N, row_ptr, sid, conprb, ncpv, theta, counts, post, post0);
#endif
}

/* EM.cpp:391-413 */
void ro_mstep(int32_t M, double* counts, double* theta, double n0, ro_round_stats* st) {
    counts[0] += n0;
    double sum = 0.0;
    for (int32_t i = 0; i <= M; ++i) sum += counts[i];
    double bchange = 0.0;
    int64_t tot = 0;
    for (int32_t i = 0; i <= M; ++i) {
        const double old = theta[i];
        const double tn = counts[i] / sum;
        if (old >= 1e-7) {
            const double change = fabs(tn - old) / old;
            if (change >= 0.001) ++tot;
            if (bchange < change) bchange = change;
        }
        theta[i] = tn;
    }
    st->sum = sum;
    st->bchange = bchange;
    st->totnum = tot;
}

int32_t ro_em_rounds(uint64_t N, const uint64_t* row_ptr, const int32_t* sid, const double* conprb,
                     const double* ncpv, int32_t M, double* theta, double n0, int32_t first_round,
                     int32_t max_rounds_this_call, int32_t min_round, int32_t max_round, ro_round_stats* stats,
                     int32_t* stopped, int32_t n_threads) {
    double* counts = (double*)malloc(sizeof(double) * ((size_t)M + 1));
    int32_t ran = 0;
    *stopped = 0;
    for (int32_t r = 0; r < max_rounds_this_call; ++r) {
        const int32_t round = first_round + r;
        ro_round_stats st;
        ro_estep(N, row_ptr, sid, conprb, ncpv, theta, M, counts, NULL, NULL, n_threads);
        ro_mstep(M, counts, theta, n0, &st);
        if (stats) stats[r] = st;
        ++ran;
        if (!(round < min_round || (st.totnum > 0 && round < max_round))) { /* EM.cpp:416 */
            *stopped = 1;
            break;
        }
    }
    free(counts);
    return ran;
}

/* ------------------------------------------------------------------------------------------ */
/* sub-model evaluation                                                                        */

/* LenDist::getAdjustedProb, LenDist.h:63-68 */
static double ld_adj(const ro_lendist* d, int len, int refL) {
    if (len <= d->lb || len > d->ub || refL <= d->lb) return 0.0;
    const int top = (d->ub < refL ? d->ub : refL) - d->lb;
    return d->pdf[len - d->lb] / d->cdf[top];
}
/* LenDist::getProb, LenDist.h:57-60 (the reference asserts the range; out of range -> 0 here) */
static double ld_prob(const ro_lendist* d, int len) {
    if (len <= d->lb || len > d->ub) return 0.0;
    return d->pdf[len - d->lb];
}
/* RSPD::evalCDF, RSPD.h:63-68 */
static double rspd_cdf_at(const ro_model* m, int fpos, int fullLen) {
    const int i = (int)(((long long)fpos) * m->rspd_B / fullLen);
    const double val = fpos * 1.0 / fullLen * m->rspd_B;
    return m->rspd_cdf[i] + (val - i) * m->rspd_pdf[i + 1];
}
/* RSPD::getAdjustedProb, RSPD.h:70-75 */
static double rspd_adj(const ro_model* m, int fpos, int effL, int fullLen) {
    if (!m->est_rspd) return 1.0 / effL;
    const double denom = rspd_cdf_at(m, effL, fullLen);
    return denom >= RO_EPS ? (rspd_cdf_at(m, fpos + 1, fullLen) - rspd_cdf_at(m, fpos, fullLen)) / denom : 0.0;
}
/* RefSeq::get_id, RefSeq.h:84-87: code of base at `p` read in direction dir */
static int ref_code(const ro_refs* rf, int sid, int p, int dir) {
    const uint8_t* s = rf->seq + rf->seq_off[sid];
    if (dir == 0) return s[p];
    const int c = s[rf->tot_len[sid] - p - 1];
    return c < 4 ? 3 - c : 4;
}
/* RefSeq::getMask, RefSeq.h:89-92 */
static int ref_mask(const ro_refs* rf, int sid, int p) {
    return (rf->mask_words[rf->mask_off[sid] + p / 32] >> (p % 32)) & 1u;
}
/* Profile::getProb (Profile.h:114-124) / QProfile::getProb (QProfile.h:111-120) */
static double seq_prob(const ro_model* m, const ro_reads* rd, int mate, uint64_t i, const ro_refs* rf, int sid, int pos,
                       int dir) {
    const uint64_t o = rd->off[mate][i];
    const int len = (int)(rd->off[mate][i + 1] - o);
    double prob = 1.0;
    if (m->model_type & 1) {
        for (int k = 0; k < len; ++k)
            prob *= m->profile[((size_t)rd->qual[mate][o + k] * 5 + ref_code(rf, sid, k + pos, dir)) * 5 + rd->base[mate][o + k]];
    } else {
        for (int k = 0; k < len; ++k)
            prob *= m->profile[((size_t)k * 5 + ref_code(rf, sid, k + pos, dir)) * 5 + rd->base[mate][o + k]];
    }
    return prob;
}
/* NoiseProfile::getProb (NoiseProfile.h:104-113) / NoiseQProfile::getProb (NoiseQProfile.h:115-124) */
static double noise_prob(const ro_model* m, const ro_reads* rd, int mate, uint64_t i) {
    const uint64_t o = rd->off[mate][i];
    const int len = (int)(rd->off[mate][i + 1] - o);
    double prob = 1.0;
    if (m->model_type & 1) {
        for (int k = 0; k < len; ++k) prob *= m->noise_profile[(size_t)rd->qual[mate][o + k] * 5 + rd->base[mate][o + k]];
    } else {
        for (int k = 0; k < len; ++k) prob *= m->noise_profile[rd->base[mate][o + k]];
    }
    return prob;
}
static int imin(int a, int b) { return a < b ? a : b; }
static int imax(int a, int b) { return a > b ? a : b; }

/* SingleModel.h:95-146 / SingleQModel.h:101-151 */
static double conprb_single(const ro_model* m, const ro_reads* rd, const ro_refs* rf, uint64_t i, int s, int pos) {
    if (rd->lowq[i]) return 0.0;
    const int sid = abs(s), dir = s < 0;
    const int fullLen = rf->full_len[sid], totLen = rf->tot_len[sid];
    const int readLen = (int)(rd->off[0][i + 1] - rd->off[0][i]);
    const int fpos = dir == 0 ? pos : totLen - pos - readLen;
    const int seedPos = dir == 0 ? pos : totLen - pos - m->seed_len;
    if (seedPos >= fullLen || ref_mask(rf, sid, seedPos)) return 0.0;
    double value;
    if (m->has_mld) {
        const int minL = imax(readLen, m->gld.lb + 1), maxL = imin(totLen - pos, m->gld.ub);
        value = 0.0;
        for (int fragLen = minL; fragLen <= maxL; ++fragLen) {
            const int pfpos = dir == 0 ? pos : totLen - pos - fragLen;
            const int effL = imin(fullLen, totLen - fragLen + 1);
            value += ld_adj(&m->gld, fragLen, totLen) * rspd_adj(m, pfpos, effL, fullLen) * ld_adj(&m->mld, readLen, fragLen);
        }
    } else {
        const int effL = imin(fullLen, totLen - readLen + 1);
        value = ld_adj(&m->gld, readLen, totLen) * rspd_adj(m, fpos, effL, fullLen);
    }
    double prob = m->ori[dir] * value * seq_prob(m, rd, 0, i, rf, sid, pos, dir);
    if (prob < RO_EPS) prob = 0.0;
    return m->mw[sid] < RO_EPS ? 0.0 : prob / m->mw[sid];
}

/* PairedEndModel.h:90-134 / PairedEndQModel.h:94-138 */
static double conprb_paired(const ro_model* m, const ro_reads* rd, const ro_refs* rf, uint64_t i, int s, int pos,
                            int insertLen) {
    if (rd->lowq[i]) return 0.0;
    const int sid = abs(s), dir = s < 0;
    const int fullLen = rf->full_len[sid], totLen = rf->tot_len[sid];
    const int fpos = dir == 0 ? pos : totLen - pos - insertLen;
    const int effL = imin(fullLen, totLen - insertLen + 1);
    if (fpos >= fullLen || ref_mask(rf, sid, fpos)) return 0.0;
    double prob = m->ori[dir] * ld_adj(&m->gld, insertLen, totLen) * rspd_adj(m, fpos, effL, fullLen);
    const int len1 = (int)(rd->off[0][i + 1] - rd->off[0][i]), len2 = (int)(rd->off[1][i + 1] - rd->off[1][i]);
    prob *= ld_adj(&m->mld, len1, insertLen) * seq_prob(m, rd, 0, i, rf, sid, pos, dir);
    const int m2pos = totLen - pos - insertLen, m2dir = !dir;
    prob *= ld_adj(&m->mld, len2, insertLen) * seq_prob(m, rd, 1, i, rf, sid, m2pos, m2dir);
    if (prob < RO_EPS) prob = 0.0;
    return m->mw[sid] < RO_EPS ? 0.0 : prob / m->mw[sid];
}

/* getNoiseConPrb: SingleQModel.h:153-162, PairedEndQModel.h:140-155 */
static double noise_conprb(const ro_model* m, const ro_reads* rd, uint64_t i) {
    if (rd->lowq[i]) return 0.0;
    double prob;
    if (m->model_type < 2) {
        const int readLen = (int)(rd->off[0][i + 1] - rd->off[0][i]);
        prob = m->has_mld ? ld_prob(&m->mld, readLen) : ld_prob(&m->gld, readLen);
        prob *= noise_prob(m, rd, 0, i);
    } else {
        const int len1 = (int)(rd->off[0][i + 1] - rd->off[0][i]), len2 = (int)(rd->off[1][i + 1] - rd->off[1][i]);
        prob = ld_prob(&m->mld, len1) * noise_prob(m, rd, 0, i);
        prob *= ld_prob(&m->mld, len2) * noise_prob(m, rd, 1, i);
    }
    if (prob < RO_EPS) prob = 0.0;
    return m->mw[0] < RO_EPS ? 0.0 : prob / m->mw[0];
}

void ro_calc_conprb(const ro_model* m, const ro_reads* rd, const ro_refs* rf, uint64_t N, const uint64_t* row_ptr,
                    const int32_t* sid, const int32_t* pos, const int32_t* insertL, double* conprb, double* ncpv) {
    for (uint64_t i = 0; i < N; ++i) { /* EM.cpp:265-275 */
        ncpv[i] = noise_conprb(m, rd, i);
        for (uint64_t j = row_ptr[i]; j < row_ptr[i + 1]; ++j)
            conprb[j] = m->model_type < 2 ? conprb_single(m, rd, rf, i, sid[j], pos[j])
                                          : conprb_paired(m, rd, rf, i, sid[j], pos[j], insertL[j]);
    }
}

/* ------------------------------------------------------------------------------------------ */
/* sufficient statistics                                                                       */

/* RSPD::update, RSPD.h:43-59 */
static void rspd_update(const ro_model* m, double* pdf, int fpos, int fullLen, double frac) {
    if (fpos >= fullLen) return;
    const int B = m->rspd_B;
    int i;
    double a = fpos * 1.0 / fullLen, b;
    for (i = (int)(((long long)fpos) * B / fullLen + 1); i < (((long long)fpos + 1) * B - 1) / fullLen + 1; ++i) {
        b = i * 1.0 / B;
        pdf[i] += (b - a) * fullLen * frac;
        a = b;
    }
    b = (fpos + 1.0) / fullLen;
    pdf[i] += (b - a) * fullLen * frac;
}
/* Profile::update (Profile.h:91-96) / QProfile::update (QProfile.h:88-93) */
static void prof_update(const ro_model* m, double* p, const ro_reads* rd, int mate, uint64_t i, const ro_refs* rf,
                        int sid, int pos, int dir, double frac) {
    const uint64_t o = rd->off[mate][i];
    const int len = (int)(rd->off[mate][i + 1] - o);
    for (int k = 0; k < len; ++k) {
        const size_t row = (m->model_type & 1) ? rd->qual[mate][o + k] : (size_t)k;
        p[(row * 5 + ref_code(rf, sid, k + pos, dir)) * 5 + rd->base[mate][o + k]] += frac;
    }
}
/* NoiseProfile::update (NoiseProfile.h:71-76) / NoiseQProfile::update (NoiseQProfile.h:74-79) */
static void noise_update(const ro_model* m, double* p, const ro_reads* rd, int mate, uint64_t i, double frac) {
    const uint64_t o = rd->off[mate][i];
    const int len = (int)(rd->off[mate][i + 1] - o);
    for (int k = 0; k < len; ++k) {
        if (m->model_type & 1) p[(size_t)rd->qual[mate][o + k] * 5 + rd->base[mate][o + k]] += frac;
        else p[rd->base[mate][o + k]] += frac;
    }
}

void ro_update_stats(const ro_model* m, const ro_reads* rd, const ro_refs* rf, uint64_t N, const uint64_t* row_ptr,
                     const int32_t* sid, const int32_t* pos, const int32_t* insertL, const double* post,
                     const double* post0, ro_model_stats* st) {
    const int hasq = m->model_type & 1, paired = m->model_type >= 2;
    memset(st->profile, 0, sizeof(double) * (hasq ? 2500 : (size_t)m->pro_len * 25));
    memset(st->noise_profile, 0, sizeof(double) * (hasq ? 500 : 5));
    if (paired) memset(st->gld_pdf, 0, sizeof(double) * ((size_t)st->gld_span + 1));
    if (m->est_rspd) memset(st->rspd_pdf, 0, sizeof(double) * ((size_t)m->rspd_B + 2));
    for (uint64_t i = 0; i < N; ++i) {
        if (rd->lowq[i]) continue; /* update/updateNoise return early for low-quality reads */
        if (post0[i] >= RO_EPS) { /* updateNoise: SingleQModel.h:217-221, PairedEndQModel.h:179-188 */
            noise_update(m, st->noise_profile, rd, 0, i, post0[i]);
            if (paired) noise_update(m, st->noise_profile, rd, 1, i, post0[i]);
        }
        for (uint64_t j = row_ptr[i]; j < row_ptr[i + 1]; ++j) {
            const double frac = post[j];
            if (frac < RO_EPS) continue;
            const int t = abs(sid[j]), dir = sid[j] < 0, p = pos[j];
            const int fullLen = rf->full_len[t], totLen = rf->tot_len[t];
            if (!paired) { /* SingleQModel.h:168-215 with mld == NULL on the helper (SURVEY A.3) */
                if (m->est_rspd) {
                    const int readLen = (int)(rd->off[0][i + 1] - rd->off[0][i]);
                    if (m->ori[0] >= 0.1 && dir == 0) rspd_update(m, st->rspd_pdf, p, fullLen, frac);
                    if (m->ori[0] < 0.1 && dir == 1) rspd_update(m, st->rspd_pdf, totLen - p - readLen, fullLen, frac);
                }
                prof_update(m, st->profile, rd, 0, i, rf, t, p, dir, frac);
            } else { /* PairedEndQModel.h:161-177 */
                const int il = insertL[j];
                if (il > st->gld_lb && il <= st->gld_lb + st->gld_span) st->gld_pdf[il - st->gld_lb] += frac; /* LenDist.h:46-49 */
                if (m->est_rspd) rspd_update(m, st->rspd_pdf, dir == 0 ? p : totLen - p - il, fullLen, frac);
                prof_update(m, st->profile, rd, 0, i, rf, t, p, dir, frac);
                prof_update(m, st->profile, rd, 1, i, rf, t, totLen - p - il, !dir, frac);
            }
        }
    }
}

/* ------------------------------------------------------------------------------------------ */
/* MT19937 (Matsumoto & Nishimura 1998; boost::random::mt19937 is this generator)             */
void ro_mt_seed(ro_mt19937* g, uint32_t seed) {
    g->mt[0] = seed;
    for (int i = 1; i < 624; ++i) g->mt[i] = 1812433253u * (g->mt[i - 1] ^ (g->mt[i - 1] >> 30)) + (uint32_t)i;
    g->idx = 624;
}
uint32_t ro_mt_next(ro_mt19937* g) {
    if (g->idx >= 624) {
        for (int k = 0; k < 624; ++k) {
            const uint32_t y = (g->mt[k] & 0x80000000u) | (g->mt[(k + 1) % 624] & 0x7fffffffu);
            g->mt[k] = g->mt[(k + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        }
        g->idx = 0;
    }
    uint32_t y = g->mt[g->idx++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
}
/* sampling.h:19-42: seeds are successive outputs of mt19937(seed), duplicates skipped */
void ro_chain_seeds(uint32_t seed, int32_t n_chains, uint32_t* out) {
    ro_mt19937 g;
    ro_mt_seed(&g, seed);
    for (int32_t c = 0; c < n_chains; ++c) {
        uint32_t s;
        int dup;
        do {
            s = ro_mt_next(&g);
            dup = 0;
            for (int32_t k = 0; k < c; ++k) if (out[k] == s) dup = 1;
        } while (dup);
        out[c] = s;
    }
}
/* uniform_01<double> over a 32-bit engine: one draw, u = x * 2^-32 (SURVEY section 8(c)) */
static double mt_uniform(ro_mt19937* g) { return ro_mt_next(g) * (1.0 / 4294967296.0); }
/* sampling.h:50-65 */
static int sample_cum(ro_mt19937* g, const double* arr, int len) {
    const double prb = mt_uniform(g) * arr[len - 1];
    int l = 0, r = len - 1;
    while (l <= r) {
        const int mid = (l + r) / 2;
        if (arr[mid] <= prb) l = mid + 1; else r = mid - 1;
    }
    return l;
}

/* WriteResults.h:55-75 */
void ro_polish_theta(int32_t M, double* theta, const double* eel, const double* mw) {
    double sum = 0.0;
    for (int32_t i = 0; i <= M; ++i) {
        if (i > 0 && (mw[i] < RO_EPS || eel[i] < RO_EPS)) { theta[i] = 0.0; continue; }
        theta[i] = theta[i] / mw[i];
        sum += theta[i];
    }
    for (int32_t i = 0; i <= M; ++i) theta[i] /= sum;
}
/* WriteResults.h:77-104 */
void ro_expression_values(int32_t M, const double* theta, const double* eel, double* tpm, double* fpkm) {
    double denom = 0.0;
    for (int32_t i = 1; i <= M; ++i) if (eel[i] >= RO_EPS) denom += theta[i];
    if (denom < RO_EPS) denom = 1.0;
    fpkm[0] = tpm[0] = 0.0;
    for (int32_t i = 1; i <= M; ++i) fpkm[i] = eel[i] >= RO_EPS ? (theta[i] / denom) * 1e9 / eel[i] : 0.0;
    denom = 0.0;
    for (int32_t i = 1; i <= M; ++i) denom += fpkm[i];
    if (denom < RO_EPS) denom = 1.0;
    for (int32_t i = 1; i <= M; ++i) tpm[i] = fpkm[i] / denom * 1e6;
}

/* Gibbs.cpp:265-353 */
void ro_gibbs_chain(uint64_t N1, const uint64_t* row_ptr, const int32_t* sid, const double* conprb, int32_t M,
                    double n0, const int32_t* init_counts, const double* pseudo_counts, double totc,
                    const double* eel, const double* mw, int32_t n_genes, const int32_t* gene_start, int32_t burnin,
                    int32_t gap, int32_t n_samples, uint32_t seed, int32_t* count_vectors, double* sum_c,
                    double* sum_c2, double* sum_tpm, double* sum_fpkm, double* sum_gene_c2) {
    ro_mt19937 g;
    ro_mt_seed(&g, seed);
    int32_t* counts = (int32_t*)malloc(sizeof(int32_t) * ((size_t)M + 1));
    int32_t* z = (int32_t*)malloc(sizeof(int32_t) * (N1 ? N1 : 1));
    double* theta = (double*)malloc(sizeof(double) * ((size_t)M + 1));
    double* tpm = (double*)malloc(sizeof(double) * ((size_t)M + 1));
    double* fpkm = (double*)malloc(sizeof(double) * ((size_t)M + 1));
    uint64_t maxlen = 1;
    for (uint64_t i = 0; i < N1; ++i) if (row_ptr[i + 1] - row_ptr[i] > maxlen) maxlen = row_ptr[i + 1] - row_ptr[i];
    double* arr = (double*)malloc(sizeof(double) * maxlen);
    memcpy(counts, init_counts, sizeof(int32_t) * ((size_t)M + 1));
    counts[0] += (int32_t)n0;
    for (uint64_t i = 0; i < N1; ++i) { /* Gibbs.cpp:281-291 */
        const uint64_t fr = row_ptr[i], len = row_ptr[i + 1] - fr;
        for (uint64_t k = 0; k < len; ++k) arr[k] = conprb[fr + k] + (k ? arr[k - 1] : 0.0);
        z[i] = sid[fr + sample_cum(&g, arr, (int)len)];
        ++counts[z[i]];
    }
    const int chainlen = 1 + (n_samples - 1) * gap;
    int kept = 0;
    for (int round = 1; round <= burnin + chainlen; ++round) {
        for (uint64_t i = 0; i < N1; ++i) { /* Gibbs.cpp:297-311 */
            --counts[z[i]];
            const uint64_t fr = row_ptr[i], len = row_ptr[i + 1] - fr;
            for (uint64_t k = 0; k < len; ++k) {
                const int t = sid[fr + k];
                arr[k] = (counts[t] + pseudo_counts[t]) * conprb[fr + k];
                if (k) arr[k] += arr[k - 1];
            }
            z[i] = sid[fr + sample_cum(&g, arr, (int)len)];
            ++counts[z[i]];
        }
        if (round > burnin && (round - burnin - 1) % gap == 0) { /* Gibbs.cpp:313-346 */
            memcpy(count_vectors + (size_t)kept * ((size_t)M + 1), counts, sizeof(int32_t) * ((size_t)M + 1));
            ++kept;
            for (int32_t i = 0; i <= M; ++i) theta[i] = counts[i] < 0 ? 0.0 : (counts[i] + pseudo_counts[i]) / totc;
            ro_polish_theta(M, theta, eel, mw);
            ro_expression_values(M, theta, eel, tpm, fpkm);
            for (int32_t i = 0; i <= M; ++i) {
                sum_c[i] += counts[i];
                sum_c2[i] += (double)counts[i] * counts[i];
                sum_tpm[i] += tpm[i];
                sum_fpkm[i] += fpkm[i];
            }
            for (int32_t gi = 0; gi < n_genes; ++gi) {
                double c = 0.0;
                for (int32_t j = gene_start[gi]; j < gene_start[gi + 1]; ++j) c += counts[j];
                sum_gene_c2[gi] += c * c;
            }
        }
    }
    free(counts); free(z); free(theta); free(tpm); free(fpkm); free(arr);
}

/* ------------------------------------------------------------------------------------------ */
/* Phase II of rsem-calculate-credibility-intervals (calcCI.cpp:218-385)                        */

/* ascending sort of n floats: LSD radix over the order-preserving unsigned image of the bits.
 * For the finite values without -0.0 that Phase I produces it orders exactly as operator<.     */
static void ci_sort(float* v, uint32_t* a, uint32_t* b, int64_t n) {
    if (n <= 32) { /* insertion sort by operator< for short rows */
        for (int64_t i = 1; i < n; ++i) {
            const float x = v[i];
            int64_t j = i;
            for (; j > 0 && x < v[j - 1]; --j) v[j] = v[j - 1];
            v[j] = x;
        }
        return;
    }
    for (int64_t i = 0; i < n; ++i) {
        uint32_t u;
        memcpy(&u, &v[i], 4);
        a[i] = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    }
    for (int shift = 0; shift < 32; shift += 8) {
        int64_t cnt[257] = {0};
        for (int64_t i = 0; i < n; ++i) ++cnt[((a[i] >> shift) & 0xff) + 1];
        for (int d = 0; d < 256; ++d) cnt[d + 1] += cnt[d];
        for (int64_t i = 0; i < n; ++i) b[cnt[(a[i] >> shift) & 0xff]++] = a[i];
        uint32_t* t = a; a = b; b = t;
    }
    for (int64_t i = 0; i < n; ++i) {
        const uint32_t u = (a[i] & 0x80000000u) ? (a[i] & 0x7fffffffu) : ~a[i];
        memcpy(&v[i], &u, 4);
    }
}

/* calcCI on s, sorted in place: out = lb, ub, cqv (calcCI.cpp:218-284) */
static void ci_calc(float* s, uint32_t* a, uint32_t* b, int n, int threshold, float* out) {
    ci_sort(s, a, b, n);
    int p = 0, q = n - 1, newp, newq = n - 1;
    /* q: the first element of the run of ties at the top that still leaves at most threshold above it */
    do {
        q = newq;
        while (newq > 0 && s[newq - 1] == s[newq]) newq--;
        newq--;
    } while (newq >= 0 && n - (newq + 1) <= threshold);
    int outside = n - (q + 1);
    float lb = (float)-1e30, ub = (float)1e30;
    do {
        const float width = s[q] - s[p], best = ub - lb;
        if (width < best) {
            lb = s[p];
            ub = s[q];
        }
        newp = p;
        while (newp < n - 1 && s[newp] == s[newp + 1]) newp++;
        newp++;
        if (newp <= threshold) {
            outside += newp - p;
            p = newp;
            while (outside > threshold && q < n - 1) {
                newq = q + 1;
                while (newq < n - 1 && s[newq] == s[newq + 1]) newq++;
                outside -= newq - q;
                q = newq;
            }
        } else {
            p = newp;
        }
    } while (p <= threshold);
    /* Tukey's hinges: a float sum halved in double, rounded back to float */
    const int quo = n / 4, res = n % 4;
    float q1, q3;
    if (res == 0) {
        const float x = s[quo - 1] + s[quo], y = s[3 * quo - 1] + s[3 * quo];
        q1 = (float)((double)x / 2.0);
        q3 = (float)((double)y / 2.0);
    } else if (res == 3) {
        const float x = s[quo] + s[quo + 1], y = s[3 * quo + 1] + s[3 * quo + 2];
        q1 = (float)((double)x / 2.0);
        q3 = (float)((double)y / 2.0);
    } else {
        q1 = s[quo];
        q3 = s[3 * quo];
    }
    const float d = q3 - q1, sum = q3 + q1;
    out[0] = lb;
    out[1] = ub;
    out[2] = d > 0.0f ? d / sum : 0.0f;
}

typedef struct ci_bufs {
    float *t, *f, *gt, *gf, *it, *itf;
    uint32_t *a, *b;
} ci_bufs;

static void ci_bufs_alloc(ci_bufs* w, int64_t n) {
    float** fs[6] = {&w->t, &w->f, &w->gt, &w->gf, &w->it, &w->itf};
    for (int i = 0; i < 6; ++i) *fs[i] = (float*)calloc((size_t)n, sizeof(float));
    w->a = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)n);
    w->b = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)n);
}

static void ci_bufs_free(ci_bufs* w) {
    free(w->t); free(w->f); free(w->gt); free(w->gf); free(w->it); free(w->itf); free(w->a); free(w->b);
}

/* an isoform ends before allele end_j (calcCI.cpp:321-330, 364-373): the running sums, sorted in place, when it has
 * several alleles, else the intervals of its one allele.  The sort happens even when the result is not kept (keep = 0):
 * the later isoforms of the range add onto the sorted sums. */
static void ci_finish_isoform(ci_bufs* w, int64_t n, int threshold, int tid, int curaid, int end_j, int keep,
                              const float* tr_out, float* iso_out) {
    float dropped[6];
    float* o = keep ? iso_out + (size_t)tid * 6 : dropped;
    if (end_j - curaid > 1) {
        ci_calc(w->it, w->a, w->b, (int)n, threshold, o);
        ci_calc(w->itf, w->a, w->b, (int)n, threshold, o + 3);
    } else {
        memcpy(o, tr_out + (size_t)(curaid - 1) * 6, 6 * sizeof(float));
    }
}

/* genes [g0, g1) with their transcripts; with isoforms, the running isoform sums of one Phase II range.  iso_last[tid]
 * is the range whose result the isoform keeps: the one holding its last allele */
static void ci_range(int64_t n, const float* samples, const float* l_bars, const int32_t* gene_start,
                     const int32_t* iso_of, const int32_t* iso_last, int32_t part, int32_t g0, int32_t g1,
                     int32_t threshold, float* tr_out, float* gene_out, float* iso_out, ci_bufs* w) {
    int curtid = -1, curaid = -1;
    if (iso_of) {
        memset(w->it, 0, sizeof(float) * (size_t)n);
        memset(w->itf, 0, sizeof(float) * (size_t)n);
    }
    for (int32_t g = g0; g < g1; ++g) {
        const int b = gene_start[g], e = gene_start[g + 1];
        memset(w->gt, 0, sizeof(float) * (size_t)n);
        memset(w->gf, 0, sizeof(float) * (size_t)n);
        for (int j = b; j < e; ++j) {
            if (iso_of && curtid != iso_of[j]) {
                if (curtid >= 0)
                    ci_finish_isoform(w, n, threshold, curtid, curaid, j, iso_last[curtid] == part, tr_out, iso_out);
                curtid = iso_of[j];
                curaid = j;
            }
            const float* row = samples + (size_t)(j - 1) * (size_t)n;
            for (int64_t k = 0; k < n; ++k) {
                w->t[k] = row[k];
                w->f[k] = (float)(1e3 / (double)l_bars[k] * (double)row[k]);
                if (iso_of) {
                    w->it[k] += w->t[k];
                    w->itf[k] += w->f[k];
                }
                w->gt[k] += w->t[k];
                w->gf[k] += w->f[k];
            }
            ci_calc(w->t, w->a, w->b, (int)n, threshold, tr_out + (size_t)(j - 1) * 6);
            ci_calc(w->f, w->a, w->b, (int)n, threshold, tr_out + (size_t)(j - 1) * 6 + 3);
        }
        if (e - b > 1) {
            ci_calc(w->gt, w->a, w->b, (int)n, threshold, gene_out + (size_t)g * 6);
            ci_calc(w->gf, w->a, w->b, (int)n, threshold, gene_out + (size_t)g * 6 + 3);
        } else {
            memcpy(gene_out + (size_t)g * 6, tr_out + (size_t)(b - 1) * 6, 6 * sizeof(float));
        }
    }
    if (iso_of && curtid >= 0)
        ci_finish_isoform(w, n, threshold, curtid, curaid, gene_start[g1], iso_last[curtid] == part, tr_out, iso_out);
}

void ro_ci_phase2(int32_t M, int64_t n, const float* samples, const float* l_bars, int32_t n_genes,
                  const int32_t* gene_start, int32_t n_isoforms, const int32_t* isoform_start, int32_t n_parts,
                  const int32_t* part_gene_start, int32_t threshold, float* tr_out, float* gene_out, float* iso_out,
                  int32_t n_threads) {
#ifdef _OPENMP
    if (n_threads < 1) n_threads = omp_get_max_threads();
#else
    n_threads = 1;
#endif
    if (n_isoforms <= 0 || !isoform_start) { /* every gene stands alone */
#ifdef _OPENMP
#pragma omp parallel num_threads(n_threads)
#endif
        {
            ci_bufs w;
            ci_bufs_alloc(&w, n);
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 16)
#endif
            for (int32_t g = 0; g < n_genes; ++g)
                ci_range(n, samples, l_bars, gene_start, NULL, NULL, 0, g, g + 1, threshold, tr_out, gene_out, NULL, &w);
            ci_bufs_free(&w);
        }
        return;
    }
    int32_t* iso_of = (int32_t*)malloc(sizeof(int32_t) * ((size_t)M + 1));
    int32_t* iso_last = (int32_t*)malloc(sizeof(int32_t) * (size_t)n_isoforms);
    int32_t* part_of = (int32_t*)malloc(sizeof(int32_t) * ((size_t)M + 1));
    for (int32_t i = 0; i < n_isoforms; ++i)
        for (int32_t j = isoform_start[i]; j < isoform_start[i + 1]; ++j) iso_of[j] = i;
    for (int32_t p = 0; p < n_parts; ++p)
        for (int32_t g = part_gene_start[p]; g < part_gene_start[p + 1]; ++g)
            for (int32_t j = gene_start[g]; j < gene_start[g + 1]; ++j) part_of[j] = p;
    for (int32_t i = 0; i < n_isoforms; ++i) iso_last[i] = part_of[isoform_start[i + 1] - 1];
#ifdef _OPENMP
#pragma omp parallel num_threads(n_threads)
#endif
    {
        ci_bufs w;
        ci_bufs_alloc(&w, n);
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 1)
#endif
        for (int32_t p = 0; p < n_parts; ++p)
            ci_range(n, samples, l_bars, gene_start, iso_of, iso_last, p, part_gene_start[p], part_gene_start[p + 1],
                     threshold, tr_out, gene_out, iso_out, &w);
        ci_bufs_free(&w);
    }
    free(iso_of); free(iso_last); free(part_of);
}
