"""bin/rsem-calculate-credibility-intervals against the reference tool (oracle/_ref/rsem-calculate-credibility-intervals,
built by oracle/ci.mk): on the count vectors of one bin/rsem-run-gibbs run, the rows both append to imd.iso_res /
imd.gene_res (and imd.allele_res) must be byte-identical, and so must stdout (with -p > 1 as a multiset of lines: the
reference's threads print in any order).  Where the reference binary is not built, its files' SHA-256 digests and
stdout come from tests/golden/reference/ci_*.tar.xz (rsem_files.reference_run; RSEM_B200_RECORD_REFERENCE=1 rewrites
them).  The reference's imd.tmp is not compared: bin/ does not write it.

Inputs are the golden data sets (all four model types): their .ofg and .model feed rsem-run-gibbs, whose count vectors
feed both tools."""
import hashlib
import os
import shutil
import subprocess
import tarfile

import pytest

import rsem_files as rf

pytestmark = pytest.mark.gpu

BIN = os.path.join(rf.ROOT, "bin", "rsem-calculate-credibility-intervals")
REF_BIN = os.path.join(rf.ROOT, "oracle", "_ref", "rsem-calculate-credibility-intervals")
RESULTS = ("s.iso_res", "s.gene_res", "s.allele_res")


def _dataset(tmp_path, key, name, nsamples, threads, seed=7, gibbs_extra=(), alleles=False):
    """a golden data set laid out as the driver leaves it, with the count vectors of one rsem-run-gibbs run"""
    d = tmp_path / key
    with tarfile.open(os.path.join(rf.ROOT, "tests", "golden", name + ".tar.gz")) as t:
        t.extractall(tmp_path / "x", filter="data")
    src = tmp_path / "x" / name
    shutil.copytree(src / "ref", d / "ref")
    os.makedirs(d / "s.temp")
    os.makedirs(d / "s.stat")
    shutil.copy(src / "s.temp" / "s.omit", d / "s.temp" / "s.omit")
    shutil.copy(src / "out" / "ofg20", d / "s.temp" / "s.ofg")
    shutil.copy(src / "out" / "model20", d / "s.stat" / "s.model")
    shutil.rmtree(tmp_path / "x")
    M = int(open(d / "ref" / "r.ti").readline().split()[0])
    if alleles:  # alleles 2k - 1 and 2k form isoform k where both lie in one gene; otherwise an allele is its own isoform
        grp = [int(x) for x in open(d / "ref" / "r.grp").read().split()]
        ta = [1]
        while ta[-1] <= M:
            a = ta[-1]
            ta.append(a + 2 if a + 1 <= M and not any(a < g <= a + 1 for g in grp) else a + 1)
        gt = [ta.index(g) for g in grp]
        open(d / "ref" / "r.ta", "w").write("\n".join(map(str, ta)) + "\n")
        open(d / "ref" / "r.gt", "w").write("\n".join(map(str, gt)) + "\n")
    extra = list(gibbs_extra)
    if "--prior" in extra:
        open(d / "prior.txt", "w").write("".join(f"{0.1 + (i % 7) * 0.4:.2f}\n" for i in range(M)))
    rf.run_gibbs(str(d), "ours", 20, nsamples, 1, threads, seed, extra=extra)
    return d


def _digests(d):
    return {f: hashlib.sha256(open(os.path.join(d, "s.temp", f), "rb").read()).hexdigest()
            for f in RESULTS if os.path.exists(os.path.join(d, "s.temp", f))}


def _compare(tmp_path, d, key, conf, ncv, nspc, threads, seed, extra=(), env=None):
    """-> our stdout; asserts identical result rows and stdout"""
    args = lambda exe: [exe, "ref/r", "s.temp/s", "s.stat/s", str(conf), str(ncv), str(nspc), "1024", "-p", str(threads),
                        "--seed", str(seed), *extra]
    ref, ours = str(tmp_path / (key + ".ref")), str(tmp_path / (key + ".ours"))
    shutil.copytree(d, ref)
    shutil.copytree(d, ours)
    r = rf.reference_run(key, ref, lambda: subprocess.run(args(REF_BIN), cwd=ref, capture_output=True, text=True),
                         digests_only=True)
    assert r.returncode == 0, r.stderr
    p = subprocess.run(args(BIN), cwd=ours, capture_output=True, text=True, env={**os.environ, **(env or {})})
    assert p.returncode == 0, p.stderr
    want = {os.path.basename(k): v for k, v in r.digests.items() if os.path.basename(k) in RESULTS}
    assert _digests(ours) == want
    if threads == 1:
        assert p.stdout == r.stdout
    else:
        assert sorted(p.stdout.splitlines()) == sorted(r.stdout.splitlines())
    return p


@pytest.mark.parametrize("name", ["se_noq", "se_q_polyA", "pe_noq", "pe_q_rspd"])
def test_model_types(tmp_path, name):
    d = _dataset(tmp_path, f"ci_{name}", name, 40, 2)
    _compare(tmp_path, d, f"ci_{name}", 0.95, 40, 25, 2, 11)


@pytest.mark.parametrize("threads,ncv,nspc", [(1, 30, 20), (2, 30, 20), (3, 30, 20), (3, 2, 200)])
def test_threads(tmp_path, threads, ncv, nspc):
    """-p 3 with nCV = 2: two samplers (rsem-run-gibbs wrote two files) and three Phase II ranges"""
    key = f"ci_p{threads}_{ncv}"
    d = _dataset(tmp_path, key, "pe_q_rspd", ncv, threads)
    _compare(tmp_path, d, key, 0.95, ncv, nspc, threads, 5)


@pytest.mark.parametrize("pc", ["1", "0.1", "0.001"])
def test_pseudo_count(tmp_path, pc):
    """0.1: the alpha < 1 branch for every transcript with no reads; 0.001: most of those draws underflow to 0, so the
    sorted rows hold long runs of ties"""
    d = _dataset(tmp_path, f"ci_pc{pc}", "se_noq", 20, 2)
    _compare(tmp_path, d, f"ci_pc{pc}", 0.95, 20, 30, 2, 3, extra=["--pseudo-count", pc])


def test_prior_upstream(tmp_path):
    d = _dataset(tmp_path, "ci_prior", "se_q_rspd", 20, 2, gibbs_extra=["--prior", "prior.txt"])
    _compare(tmp_path, d, "ci_prior", 0.95, 20, 30, 2, 8)


@pytest.mark.parametrize("nspc", [1, 2, 3, 4])
def test_sample_count_residues(tmp_path, nspc):
    """41 count vectors: nSamples % 4 = 1, 2, 3, 0 (the four branches of Tukey's hinges)"""
    d = _dataset(tmp_path, f"ci_r{nspc}", "pe_noq", 41, 1)
    _compare(tmp_path, d, f"ci_r{nspc}", 0.95, 41, nspc, 1, 2)


def test_confidence_half(tmp_path):
    d = _dataset(tmp_path, "ci_c50", "se_q_polyA", 20, 2)
    _compare(tmp_path, d, "ci_c50", 0.5, 20, 50, 2, 4)


def test_allele_specific_reference(tmp_path):
    """.ta / .gt: transcript rows go to imd.allele_res, isoform rows to imd.iso_res.  -p 1: the reference's isoform sums
    run on across isoforms in sample order, which with several samplers depends on their timing"""
    d = _dataset(tmp_path, "ci_allele", "se_q_rspd", 20, 1, alleles=True)
    _compare(tmp_path, d, "ci_allele", 0.95, 20, 30, 1, 9)
    assert os.path.exists(tmp_path / "ci_allele.ours" / "s.temp" / "s.allele_res")


def test_blocked_path(tmp_path):
    """a device budget far below the sample matrix: rows stay in pinned host memory, blocks of a few genes"""
    d = _dataset(tmp_path, "ci_blocked", "pe_q_rspd", 40, 2)
    n, M = 40 * 25, int(open(d / "ref" / "r.ti").readline().split()[0])
    grp = [int(x) for x in open(d / "ref" / "r.grp").read().split()]
    rows = max(2 * (b - a) + (2 if b - a > 1 else 0) for a, b in zip(grp, grp[1:]))
    budget = n * M * 2 + n * 20 + (1 << 20) + rows * n * 12   # half the sample matrix + the largest gene's rows
    p = _compare(tmp_path, d, "ci_blocked", 0.95, 40, 25, 2, 11,
                 env={"RSEM_B200_CI_DEVICE_BYTES": str(budget), "RSEM_B200_TIMING": "1"})
    assert "sample matrix in host memory" in p.stderr and " 1 blocks" not in p.stderr


def test_two_seeds(tmp_path):
    d = _dataset(tmp_path, "ci_seeds", "pe_noq", 20, 2)
    a = _compare(tmp_path, d, "ci_seed1", 0.95, 20, 30, 2, 1)
    b = _compare(tmp_path, d, "ci_seed2", 0.95, 20, 30, 2, 2)
    assert a.stdout == b.stdout
    assert _digests(tmp_path / "ci_seed1.ours") != _digests(tmp_path / "ci_seed2.ours")


def _max_gene_rows(d):
    grp = [int(x) for x in open(d / "ref" / "r.grp").read().split()]
    return max(2 * (b - a) + (2 if b - a > 1 else 0) for a, b in zip(grp, grp[1:]))


def test_resident_matrix_several_blocks(tmp_path):
    """the sample matrix fits on the device, the blocks of rows after it hold a few genes each"""
    d = _dataset(tmp_path, "ci_blocked", "pe_q_rspd", 40, 2)
    n, M = 40 * 25, int(open(d / "ref" / "r.ti").readline().split()[0])
    budget = n * M * 4 + n * 20 + (1 << 20) + 3 * _max_gene_rows(d) * n * 8
    p = _compare(tmp_path, d, "ci_blocked", 0.95, 40, 25, 2, 11,
                 env={"RSEM_B200_CI_DEVICE_BYTES": str(budget), "RSEM_B200_TIMING": "1"})
    assert "sample matrix on the device" in p.stderr and " 1 blocks" not in p.stderr


def test_allele_specific_blocked(tmp_path):
    """the running isoform sums carried from one block to the next (matrix in host memory, blocks of a few genes)"""
    d = _dataset(tmp_path, "ci_allele", "se_q_rspd", 20, 1, alleles=True)
    n, M = 20 * 30, int(open(d / "ref" / "r.ti").readline().split()[0])
    budget = n * 20 + (1 << 20) + _max_gene_rows(d) * n * 12 + n * 4   # the largest gene's rows, not the matrix
    p = _compare(tmp_path, d, "ci_allele", 0.95, 20, 30, 1, 9,
                 env={"RSEM_B200_CI_DEVICE_BYTES": str(budget), "RSEM_B200_TIMING": "1"})
    assert "sample matrix in host memory" in p.stderr and " 1 blocks" not in p.stderr
