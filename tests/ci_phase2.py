"""Host-side rules of rsem-calculate-credibility-intervals' Phase II, restated for the tests of K8 (ci_kernels.cu), and
a run of the reference tool that leaves its transcript-major sample file behind.

- parts(): the gene ranges of the reference's Phase II threads for -p threads (calcCI.cpp:402-420, main_ci.cpp).
- block_rule() / blocks(): how ci_begin / ci_end size the device work.  fixed = 20 n + 1 MiB (l_bars, the isoform sums
  and their sort buffers, small arrays); per_row = 8 n bytes with the sample matrix S on the device (the rows and
  CUB's alternate buffer) or 12 n with S in pinned host memory (plus the column staging).  S is resident iff
  budget >= S + fixed + max_rows * 8 n; rows_cap = min((budget - S_resident - fixed) // per_row, INT32_MAX // n,
  all_rows); blocks are filled greedily with whole genes."""
import os
import shutil
import subprocess
import tarfile

import numpy as np

import rsem_files as rf

INT32_MAX = 2**31 - 1
REF_BIN = os.path.join(rf.ROOT, "oracle", "_ref", "rsem-calculate-credibility-intervals")


def threshold(confidence, n):
    return n - (int(confidence * n - 1e-8) + 1)


def parts(gene_start, threads):
    M, m = gene_start[-1] - 1, len(gene_start) - 1
    n_parts, quotient = threads, M // threads
    if quotient < 1:
        n_parts, quotient = M, 1
    out, cur = [0], 0
    for i in range(n_parts):
        num = 0
        while m - cur > n_parts - i - 1 and (i == n_parts - 1 or num < quotient):
            num += gene_start[cur + 1] - gene_start[cur]
            cur += 1
        out.append(cur)
    return out


def gene_rows(gene_start):
    w = np.diff(np.asarray(gene_start, np.int64))
    return 2 * w + 2 * (w > 1)


def block_rule(gene_start, n, budget):
    """-> (resident, rows_cap, max_rows, all_rows)"""
    rows = gene_rows(gene_start)
    M = gene_start[-1] - 1
    s_bytes, fixed = 4 * n * M, 20 * n + (1 << 20)
    max_rows, all_rows = int(rows.max()), int(rows.sum())
    resident = budget >= s_bytes + fixed + max_rows * 8 * n
    per_row = 8 * n if resident else 12 * n
    rows_cap = min((budget - (s_bytes if resident else 0) - fixed) // per_row, INT32_MAX // n, all_rows)
    return resident, rows_cap, max_rows, all_rows


def blocks(gene_start, rows_cap):
    """rows of each block of genes, filled greedily"""
    out, cur = [], 0
    for r in gene_rows(gene_start):
        if cur + r > rows_cap:
            out.append(cur)
            cur = 0
        cur += int(r)
    return out + [cur]


def write_allele_tables(refdir, M):
    """.ta / .gt: alleles 2k - 1 and 2k form isoform k where both lie in one gene; otherwise an allele is its own
    isoform"""
    grp = [int(x) for x in open(os.path.join(refdir, "r.grp")).read().split()]
    ta = [1]
    while ta[-1] <= M:
        a = ta[-1]
        ta.append(a + 2 if a + 1 <= M and not any(a < g <= a + 1 for g in grp) else a + 1)
    gt = [ta.index(g) for g in grp]
    open(os.path.join(refdir, "r.ta"), "w").write("\n".join(map(str, ta)) + "\n")
    open(os.path.join(refdir, "r.gt"), "w").write("\n".join(map(str, gt)) + "\n")
    return ta


def reference_run(tmp_path, threads, nspc, alleles=False, confidence=0.95, seed=13):
    """the reference tool on the pe_noq golden set's own count vectors (2 files of 3; with -p 1 it reads the first
    only, so nCV is 3): -> dict with the data set's directory, M, gene_start, isoform_start (or None), nSamples, the
    samples it left in imd.tmp (M x nSamples, transcript-major) and the 6 rows it appended to each result file"""
    with tarfile.open(os.path.join(rf.ROOT, "tests", "golden", "pe_noq.tar.gz")) as t:
        t.extractall(tmp_path, filter="data")
    d = tmp_path / "pe_noq"
    for i in range(2):
        shutil.copy(d / "out" / f"countvectors{i}", d / "s.temp" / f"s.countvectors{i}")
    shutil.copy(d / "out" / "model20", d / "s.stat" / "s.model")
    M = int(open(d / "ref" / "r.ti").readline().split()[0])
    gene_start = [int(x) for x in open(d / "ref" / "r.grp").read().split()]
    iso = write_allele_tables(d / "ref", M) if alleles else None
    ncv = 3 * min(threads, 2)
    n = ncv * nspc
    p = subprocess.run([REF_BIN, "ref/r", "s.temp/s", "s.stat/s", str(confidence), str(ncv), str(nspc), "1024", "-p",
                        str(threads), "--seed", str(seed), "-q"], cwd=d, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    samples = np.fromfile(d / "s.temp" / "s.tmp", np.float32)
    assert samples.size == M * n
    rows = {f: open(d / "s.temp" / f).read().splitlines()[-6:]
            for f in ("s.iso_res", "s.gene_res", "s.allele_res") if os.path.exists(d / "s.temp" / f)}
    return dict(dir=d, M=M, gene_start=gene_start, isoform_start=iso, n=n, samples=samples.reshape(M, n), rows=rows,
                threshold=threshold(confidence, n), parts=parts(gene_start, threads))


def text_rows(values):
    """lb, ub, cqv columns (items x 3) as the reference prints them: %.6g, tab-separated, one line per column"""
    return ["\t".join("%.6g" % float(x) for x in values[:, c]) for c in range(3)]
