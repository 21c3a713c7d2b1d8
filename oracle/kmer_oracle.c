/* TEST INFRASTRUCTURE ONLY.  A plain-C restatement of the counts rsem-for-ebseq-calculate-clustering-info computes
 * (EBSeq/calcClusteringInfo.cpp:101-130), the way the reference computes them: one record per k-mer start, sorted by
 * the k bases and then the transcript, and one pass over the groups of equal k-mers.  The tests check
 * rsem_b200_kmer_shared (K9) against it where running the reference binary is inconvenient (forced passes, small
 * fingerprints).  Built into oracle/libkmer_oracle.so by oracle/ebseq.mk; nothing under rsem_b200/ uses it.
 *
 * Transcript t (0-based) is bases[off[t] .. off[t + 1]), codes 0..4 (A C G T N).  counts[t] receives the number of start
 * positions of t whose k-mer group holds another transcript.  k <= 0 behaves as in the reference: len - k + 1 positions
 * per transcript and a comparator that compares no bases.  Returns 0, or -1 when memory runs out.  Not thread-safe. */
#include <stdint.h>
#include <stdlib.h>

typedef struct {
    uint32_t tid;
    uint64_t pos; /* global position of the k-mer's first base */
} Cand;

static const uint8_t* g_bases;
static int g_k;

static int cand_cmp(const void* pa, const void* pb) {
    const Cand* a = (const Cand*)pa;
    const Cand* b = (const Cand*)pb;
    for (int i = 0; i < g_k; i++) {
        const uint8_t x = g_bases[a->pos + i], y = g_bases[b->pos + i];
        if (x != y) return x < y ? -1 : 1;
    }
    return a->tid < b->tid ? -1 : (a->tid > b->tid ? 1 : 0);
}

static int seq_equal(const Cand* a, const Cand* b) {
    for (int i = 0; i < g_k; i++)
        if (g_bases[a->pos + i] != g_bases[b->pos + i]) return 0;
    return 1;
}

int ko_shared_counts(int32_t k, uint64_t n, const uint64_t* off, const uint8_t* bases, uint64_t* counts) {
    uint64_t total = 0;
    for (uint64_t t = 0; t < n; t++) {
        const int64_t effL = (int64_t)(off[t + 1] - off[t]) - k + 1;
        counts[t] = 0;
        if (effL > 0) total += (uint64_t)effL;
    }
    Cand* c = (Cand*)malloc((total ? total : 1) * sizeof(Cand));
    if (!c) return -1;
    uint64_t m = 0;
    for (uint64_t t = 0; t < n; t++) {
        const int64_t effL = (int64_t)(off[t + 1] - off[t]) - k + 1;
        for (int64_t j = 0; j < effL; j++) {
            c[m].tid = (uint32_t)t;
            c[m].pos = off[t] + (uint64_t)j;
            m++;
        }
    }
    g_bases = bases;
    g_k = k;
    qsort(c, m, sizeof(Cand), cand_cmp);
    uint64_t p = 0;
    for (uint64_t i = 1; i <= m; i++) {
        if (i < m && seq_equal(&c[p], &c[i])) continue;
        const uint64_t denominator = i - p;
        uint64_t q = p;
        for (uint64_t j = p + 1; j <= i; j++)
            if (j == i || c[q].tid != c[j].tid) {
                if (j - q < denominator) counts[c[q].tid] += j - q;
                q = j;
            }
        p = i;
    }
    free(c);
    return 0;
}
