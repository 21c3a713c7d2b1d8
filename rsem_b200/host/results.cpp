// Result tables: imd.iso_res / imd.gene_res (/ imd.allele_res) written by rsem-run-em and appended to
// by rsem-run-gibbs.  Row-major TSV, one row per output column; the Perl driver transposes them
// (rsem_perl_utils.pm:44-90).  Semantics: WriteResults.h:125-479.
#include <cmath>
#include <cstring>

#include "host.hpp"

namespace host {

namespace {

struct Row {
    FILE* fo;
    explicit Row(FILE* f) : fo(f) {}
    template <class F>
    void cells(int first, int last, F&& cell) {  // inclusive range, tab separated, newline at the end
        for (int i = first; i <= last; ++i) {
            cell(i);
            fputc(i < last ? '\t' : '\n', fo);
        }
    }
    void doubles(const std::vector<double>& v, int first, int last, double scale = 1.0) {
        cells(first, last, [&](int i) { fprintf(fo, "%.2f", v[i] * scale); });
    }
};

FILE* open_or_die(const std::string& path, const char* mode) {
    FILE* f = fopen(path.c_str(), mode);
    if (!f) die("Cannot open " + path + "!");
    return f;
}

// per-group sums + within-group percentages shared by the gene and the allele/"trans" levels
struct GroupAgg {
    std::vector<double> lens, eels, counts, tpm, fpkm;
};

void aggregate(const std::vector<int>& starts, const std::vector<double>& tlens, const std::vector<double>& eel,
               const double* counts, const std::vector<double>& tpm, const std::vector<double>& fpkm, GroupAgg& g,
               std::vector<double>& pct) {
    const int m = (int)starts.size() - 1;
    g.lens.assign(m, 0.0); g.eels.assign(m, 0.0); g.counts.assign(m, 0.0); g.tpm.assign(m, 0.0); g.fpkm.assign(m, 0.0);
    for (int i = 0; i < m; ++i) {
        const int b = starts[i], e = starts[i + 1];
        for (int j = b; j < e; ++j) {
            g.counts[i] += counts[j];
            g.tpm[i] += tpm[j];
            g.fpkm[i] += fpkm[j];
        }
        if (g.tpm[i] < kEps) {  // unexpressed group: plain averages (WriteResults.h:170-176)
            const double frac = 1.0 / (e - b);
            for (int j = b; j < e; ++j) {
                g.lens[i] += tlens[j] * frac;
                g.eels[i] += eel[j] * frac;
            }
        } else {
            for (int j = b; j < e; ++j) {
                pct[j] = g.tpm[i] > kEps ? tpm[j] / g.tpm[i] : 0.0;
                g.lens[i] += tlens[j] * pct[j];
                g.eels[i] += eel[j] * pct[j];
            }
        }
    }
}

}  // namespace

void write_results_em(const std::string& ref_name, const std::string& imd_name, const std::vector<TranscriptInfo>& tr,
                      const std::vector<double>& theta, const std::vector<double>& eel, const double* counts,
                      bool append_names) {
    const int M = (int)theta.size() - 1;
    std::vector<int> gi, gt, ta;
    load_groups(ref_name + ".grp", gi);
    const int m = (int)gi.size() - 1;
    const bool alleleS = load_allele_groups(ref_name, gt, ta);

    std::vector<double> tpm, fpkm;
    expression_values(theta, eel, tpm, fpkm);
    std::vector<double> tlens(M + 1, 0.0), isopct(M + 1, 0.0);
    for (int j = 1; j <= M; ++j) tlens[j] = tr[j].length;
    GroupAgg gene;
    aggregate(gi, tlens, eel, counts, tpm, fpkm, gene, isopct);

    auto id_with_name = [&](FILE* fo, const std::string& id, const std::string& name) {
        fprintf(fo, "%s", id.c_str());
        if (append_names && name != "") fprintf(fo, "_%s", name.c_str());
    };
    std::vector<double> cnt(counts, counts + M + 1);

    if (!alleleS) {
        FILE* fo = open_or_die(imd_name + ".iso_res", "w");
        Row r(fo);
        r.cells(1, M, [&](int i) { id_with_name(fo, tr[i].transcript_id, tr[i].transcript_name); });
        r.cells(1, M, [&](int i) { id_with_name(fo, tr[i].gene_id, tr[i].gene_name); });
        r.cells(1, M, [&](int i) { fprintf(fo, "%d", tr[i].length); });
        r.doubles(eel, 1, M);
        r.doubles(cnt, 1, M);
        r.doubles(tpm, 1, M);
        r.doubles(fpkm, 1, M);
        r.doubles(isopct, 1, M, 1e2);
        fclose(fo);
    } else {
        const int m_trans = (int)ta.size() - 1;
        std::vector<double> ta_pct(M + 1, 0.0), gt_pct(m_trans, 0.0);
        GroupAgg trans;
        aggregate(ta, tlens, eel, counts, tpm, fpkm, trans, ta_pct);
        for (int i = 0; i < m; ++i)
            if (gene.tpm[i] >= kEps)
                for (int j = gt[i]; j < gt[i + 1]; ++j) gt_pct[j] = gene.tpm[i] > kEps ? trans.tpm[j] / gene.tpm[i] : 0.0;

        FILE* fo = open_or_die(imd_name + ".allele_res", "w");
        Row r(fo);
        r.cells(1, M, [&](int i) { fprintf(fo, "%s", tr[i].seqname.c_str()); });
        r.cells(1, M, [&](int i) { fprintf(fo, "%s", tr[i].transcript_id.c_str()); });
        r.cells(1, M, [&](int i) { fprintf(fo, "%s", tr[i].gene_id.c_str()); });
        r.cells(1, M, [&](int i) { fprintf(fo, "%d", tr[i].length); });
        r.doubles(eel, 1, M);
        r.doubles(cnt, 1, M);
        r.doubles(tpm, 1, M);
        r.doubles(fpkm, 1, M);
        r.doubles(ta_pct, 1, M, 1e2);
        r.doubles(isopct, 1, M, 1e2);
        fclose(fo);

        fo = open_or_die(imd_name + ".iso_res", "w");
        Row r2(fo);
        r2.cells(0, m_trans - 1, [&](int i) { fprintf(fo, "%s", tr[ta[i]].transcript_id.c_str()); });
        r2.cells(0, m_trans - 1, [&](int i) { fprintf(fo, "%s", tr[ta[i]].gene_id.c_str()); });
        r2.doubles(trans.lens, 0, m_trans - 1);
        r2.doubles(trans.eels, 0, m_trans - 1);
        r2.doubles(trans.counts, 0, m_trans - 1);
        r2.doubles(trans.tpm, 0, m_trans - 1);
        r2.doubles(trans.fpkm, 0, m_trans - 1);
        r2.doubles(gt_pct, 0, m_trans - 1, 1e2);
        fclose(fo);
    }

    FILE* fo = open_or_die(imd_name + ".gene_res", "w");
    Row r(fo);
    r.cells(0, m - 1, [&](int i) { id_with_name(fo, tr[gi[i]].gene_id, tr[gi[i]].gene_name); });
    r.cells(0, m - 1, [&](int i) {  // comma separated list of the gene's distinct transcript ids
        std::string cur;
        for (int j = gi[i]; j < gi[i + 1]; ++j) {
            if (cur != tr[j].transcript_id) {
                if (cur != "") fputc(',', fo);
                id_with_name(fo, tr[j].transcript_id, tr[j].transcript_name);
                cur = tr[j].transcript_id;
            }
        }
    });
    r.doubles(gene.lens, 0, m - 1);
    r.doubles(gene.eels, 0, m - 1);
    r.doubles(gene.counts, 0, m - 1);
    r.doubles(gene.tpm, 0, m - 1);
    r.doubles(gene.fpkm, 0, m - 1);
    fclose(fo);
    if (g_verbose) printf("Expression Results are written!\n");
}

void write_results_gibbs(const std::string& ref_name, const std::string& imd_name, int M, const std::vector<double>& pme_c,
                         const std::vector<double>& pme_fpkm, const std::vector<double>& pme_tpm,
                         const std::vector<double>& pve_c, const std::vector<double>& pve_c_genes,
                         const std::vector<double>& pve_c_trans) {
    std::vector<int> gi, gt, ta;
    load_groups(ref_name + ".grp", gi);
    const int m = (int)gi.size() - 1;
    const bool alleleS = load_allele_groups(ref_name, gt, ta);
    const int m_trans = alleleS ? (int)ta.size() - 1 : 0;

    std::vector<double> isopct(M + 1, 0.0), gene_counts(m, 0.0), gene_tpm(m, 0.0), gene_fpkm(m, 0.0);
    for (int i = 0; i < m; ++i) {
        for (int j = gi[i]; j < gi[i + 1]; ++j) {
            gene_counts[i] += pme_c[j];
            gene_tpm[i] += pme_tpm[j];
            gene_fpkm[i] += pme_fpkm[j];
        }
        if (gene_tpm[i] < kEps) continue;
        for (int j = gi[i]; j < gi[i + 1]; ++j) isopct[j] = pme_tpm[j] / gene_tpm[i];
    }
    std::vector<double> sd_c(M + 1), sd_g(m), sd_t(m_trans);
    for (int i = 0; i <= M; ++i) sd_c[i] = sqrt(pve_c[i]);
    for (int i = 0; i < m; ++i) sd_g[i] = sqrt(pve_c_genes[i]);

    if (!alleleS) {
        FILE* fo = open_or_die(imd_name + ".iso_res", "a");
        Row r(fo);
        r.doubles(pme_c, 1, M);
        r.doubles(sd_c, 1, M);
        r.doubles(pme_tpm, 1, M);
        r.doubles(pme_fpkm, 1, M);
        r.doubles(isopct, 1, M, 1e2);
        fclose(fo);
    } else {
        std::vector<double> ta_pct(M + 1, 0.0), gt_pct(m_trans, 0.0), tc(m_trans, 0.0), tt(m_trans, 0.0), tf(m_trans, 0.0);
        for (int i = 0; i < m_trans; ++i) {
            for (int j = ta[i]; j < ta[i + 1]; ++j) { tc[i] += pme_c[j]; tt[i] += pme_tpm[j]; tf[i] += pme_fpkm[j]; }
            if (tt[i] < kEps) continue;
            for (int j = ta[i]; j < ta[i + 1]; ++j) ta_pct[j] = pme_tpm[j] / tt[i];
            sd_t[i] = 0;
        }
        for (int i = 0; i < m_trans; ++i) sd_t[i] = sqrt(pve_c_trans[i]);
        for (int i = 0; i < m; ++i)
            if (gene_tpm[i] >= kEps)
                for (int j = gt[i]; j < gt[i + 1]; ++j) gt_pct[j] = tt[j] / gene_tpm[i];
        FILE* fo = open_or_die(imd_name + ".allele_res", "a");
        Row r(fo);
        r.doubles(pme_c, 1, M);
        r.doubles(sd_c, 1, M);
        r.doubles(pme_tpm, 1, M);
        r.doubles(pme_fpkm, 1, M);
        r.doubles(ta_pct, 1, M, 1e2);
        r.doubles(isopct, 1, M, 1e2);
        fclose(fo);
        fo = open_or_die(imd_name + ".iso_res", "a");
        Row r2(fo);
        r2.doubles(tc, 0, m_trans - 1);
        r2.doubles(sd_t, 0, m_trans - 1);
        r2.doubles(tt, 0, m_trans - 1);
        r2.doubles(tf, 0, m_trans - 1);
        r2.doubles(gt_pct, 0, m_trans - 1, 1e2);
        fclose(fo);
    }
    FILE* fo = open_or_die(imd_name + ".gene_res", "a");
    Row r(fo);
    r.doubles(gene_counts, 0, m - 1);
    r.doubles(sd_g, 0, m - 1);
    r.doubles(gene_tpm, 0, m - 1);
    r.doubles(gene_fpkm, 0, m - 1);
    fclose(fo);
    if (g_verbose) printf("Gibbs based expression values are written!\n");
}

}  // namespace host

namespace host {

// writeResultsSimulation (WriteResults.h:481-635): one row per transcript / gene, from the simulated counts
void write_results_simulation(const std::string& ref_name, const std::string& out_name,
                              const std::vector<TranscriptInfo>& tr, const std::vector<double>& eel,
                              const std::vector<double>& counts) {
    const int M = (int)counts.size() - 1;
    std::vector<int> gi, gt, ta;
    load_groups(ref_name + ".grp", gi);
    const int m = (int)gi.size() - 1;
    const bool alleleS = load_allele_groups(ref_name, gt, ta);
    for (int i = 1; i <= M; ++i)
        if (!(eel[i] > kEps || counts[i] <= kEps)) die("An isoform whose effecitve length < 1.000000 got sampled!");

    std::vector<double> tpm, fpkm;
    expression_values(counts, eel, tpm, fpkm);
    std::vector<double> tlens(M + 1, 0.0), isopct(M + 1, 0.0);
    for (int j = 1; j <= M; ++j) tlens[j] = tr[j].length;
    GroupAgg gene;
    aggregate(gi, tlens, eel, counts.data(), tpm, fpkm, gene, isopct);

    if (alleleS) {
        const int m_trans = (int)ta.size() - 1;
        std::vector<double> ta_pct(M + 1, 0.0), gt_pct(m_trans, 0.0);
        GroupAgg trans;
        aggregate(ta, tlens, eel, counts.data(), tpm, fpkm, trans, ta_pct);
        for (int i = 0; i < m; ++i)
            if (gene.tpm[i] >= kEps)
                for (int j = gt[i]; j < gt[i + 1]; ++j) gt_pct[j] = trans.tpm[j] / gene.tpm[i];

        FILE* fo = open_or_die(out_name + ".sim.alleles.results", "w");
        fprintf(fo, "allele_id\ttranscript_id\tgene_id\tlength\teffective_length\tcount\tTPM\tFPKM\tAlleleIsoPct\tAlleleGenePct\n");
        for (int i = 1; i <= M; ++i)
            fprintf(fo, "%s\t%s\t%s\t%d\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\n", tr[i].seqname.c_str(),
                    tr[i].transcript_id.c_str(), tr[i].gene_id.c_str(), tr[i].length, eel[i], counts[i], tpm[i], fpkm[i],
                    ta_pct[i] * 1e2, isopct[i] * 1e2);
        fclose(fo);

        fo = open_or_die(out_name + ".sim.isoforms.results", "w");
        fprintf(fo, "transcript_id\tgene_id\tlength\teffective_length\tcount\tTPM\tFPKM\tIsoPct\n");
        for (int i = 0; i < m_trans; ++i) {
            const TranscriptInfo& t = tr[ta[i]];
            fprintf(fo, "%s\t%s\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\n", t.transcript_id.c_str(), t.gene_id.c_str(),
                    trans.lens[i], trans.eels[i], trans.counts[i], trans.tpm[i], trans.fpkm[i], gt_pct[i] * 1e2);
        }
        fclose(fo);
    } else {
        FILE* fo = open_or_die(out_name + ".sim.isoforms.results", "w");
        fprintf(fo, "transcript_id\tgene_id\tlength\teffective_length\tcount\tTPM\tFPKM\tIsoPct\n");
        for (int i = 1; i <= M; ++i)
            fprintf(fo, "%s\t%s\t%d\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\n", tr[i].transcript_id.c_str(), tr[i].gene_id.c_str(),
                    tr[i].length, eel[i], counts[i], tpm[i], fpkm[i], isopct[i] * 1e2);
        fclose(fo);
    }

    FILE* fo = open_or_die(out_name + ".sim.genes.results", "w");
    fprintf(fo, "gene_id\ttranscript_id(s)\tlength\teffective_length\tcount\tTPM\tFPKM\n");
    for (int i = 0; i < m; ++i) {
        fprintf(fo, "%s\t", tr[gi[i]].gene_id.c_str());
        std::string cur;
        for (int j = gi[i]; j < gi[i + 1]; ++j)
            if (cur != tr[j].transcript_id) {
                if (cur != "") fputc(',', fo);
                fputs(tr[j].transcript_id.c_str(), fo);
                cur = tr[j].transcript_id;
            }
        fprintf(fo, "\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\n", gene.lens[i], gene.eels[i], gene.counts[i], gene.tpm[i], gene.fpkm[i]);
    }
    fclose(fo);
}

}  // namespace host
