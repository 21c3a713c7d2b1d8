"""bin/rsem-simulate-reads against the reference simulator (oracle/_ref/rsem-simulate-reads, built by
oracle/simulate.mk): for the same --seed every output file and the stdout lines must be byte-identical.  Where the
reference binary is not built, its outputs' SHA-256 digests and stdout come from tests/golden/reference/sim_*.tar.xz
(rsem_files.reference_run); RSEM_B200_RECORD_REFERENCE=1 rewrites them, and with RSEM_B200_SIM_RECORD_ONLY=1 only the
reference side runs (to record them on a machine without a GPU).

Inputs are the .model files and references of the golden data sets (all four model types, estRSPD 0 and 1, a
poly(A) reference), edited copies of them, and results files the test writes with chosen TPMs, some of them 0."""
import hashlib
import os
import random
import re
import shutil
import subprocess
import tarfile

import pytest

import rsem_files as rf

pytestmark = pytest.mark.gpu

BIN = os.path.join(rf.ROOT, "bin", "rsem-simulate-reads")
REF_BIN = os.path.join(rf.ROOT, "oracle", "_ref", "rsem-simulate-reads")
SETS = ["se_noq", "se_q_polyA", "pe_noq", "pe_q_rspd", "se_q_rspd"]  # model types 0, 1, 2, 3, 1 (estRSPD)
RECORD_ONLY = os.environ.get("RSEM_B200_SIM_RECORD_ONLY") == "1"


def _golden(tmp_path, name):
    g = tmp_path / ("golden_" + name)
    if not g.exists():
        g.mkdir()
        with tarfile.open(os.path.join(rf.ROOT, "tests", "golden", name + ".tar.gz")) as t:
            t.extractall(g, filter="data")
    return g / name


def _results(path, M, extra_col=False, rows=None, final_newline=True):
    rng = random.Random(7)
    lines = ["transcript_id\tgene_id\tlength\teffective_length\texpected_count\tTPM\tFPKM\tIsoPct"]
    for i in range(1, M + 1):
        tpm = 0.0 if i % 7 == 0 else rng.uniform(0, 100)
        lines.append(f"T{i}\tG\t1\t1\t1\t" + ("1\t" if extra_col else "") + f"{tpm:.2f}\t0\t0")
    if rows is not None:
        lines = lines[:rows + 1]
    open(path, "w").write("\n".join(lines) + ("\n" if final_newline else ""))


def _case(tmp_path, key, name, model_lines=None, **res_kw):
    """a directory holding exactly the inputs of one run: ref/, model, res.tsv"""
    src = _golden(tmp_path, name)
    d = tmp_path / key
    shutil.copytree(src / "ref", d / "ref")
    lines = open(src / "out" / "model20").read().split("\n")
    open(d / "model", "w").write("\n".join(model_lines(lines) if model_lines else lines))
    M = int(open(d / "ref" / "r.ti").readline().split()[0])
    _results(d / "res.tsv", M, **res_kw)
    return d


def _digests(out):
    return {f: hashlib.sha256(open(os.path.join(out, f), "rb").read()).hexdigest() for f in sorted(os.listdir(out))}


def _compare(d, key, theta0, n, seed, env=None):
    """-> the reference's stdout; asserts that bin/rsem-simulate-reads writes the same files and stdout"""
    args = lambda exe, out: [exe, str(d / "ref" / "r"), str(d / "model"), str(d / "res.tsv"), str(theta0), str(n),
                             os.path.join(out, "s"), "--seed", str(seed)]
    env = {**os.environ, **(env or {})}
    o_ref, o_gpu = str(d) + ".ref", str(d) + ".gpu"
    for o in (o_ref, o_gpu):
        shutil.rmtree(o, ignore_errors=True)
        os.makedirs(o)
    ref = rf.reference_run(key, str(d), lambda: subprocess.run(args(REF_BIN, o_ref), capture_output=True, text=True, env=env),
                           out=o_ref, digests_only=True)
    assert ref.returncode == 0, ref.stderr
    if RECORD_ONLY:
        return ref.stdout
    p = subprocess.run(args(BIN, o_gpu), capture_output=True, text=True, env=env)
    assert p.returncode == 0, p.stderr
    assert _digests(o_gpu) == ref.digests
    assert p.stdout == ref.stdout
    return ref.stdout


def _resim(stdout):
    return int(re.search(r"Total number of resimulation is (\d+)", stdout).group(1))


@pytest.mark.parametrize("name", SETS)
@pytest.mark.parametrize("theta0", [0.0, 0.2])
def test_identical_to_reference(tmp_path, name, theta0):
    d = _case(tmp_path, f"sim_{name}_{theta0}", name)
    _compare(d, f"sim_{name}_{theta0}", theta0, 3000, 11)


@pytest.mark.parametrize("name", ["pe_q_rspd", "se_noq"])
def test_many_windows(tmp_path, name):
    """a window of a few thousand words: attempts and reads straddle many window bounds"""
    d = _case(tmp_path, f"sim_win_{name}", name)
    _compare(d, f"sim_win_{name}", 0.1, 20000, 5, env={"RSEM_B200_SIM_WINDOW": "3000"})


def test_million_reads_gen_lines(tmp_path):
    d = _case(tmp_path, "sim_1m", "se_noq")
    assert "GEN 1000000" in _compare(d, "sim_1m", 0.05, 1000000, 3)


def _zero_rspd_bins(lines):
    """estRSPD with its first 14 of 20 bins 0: RSPD::simulate fails (no draw) whenever evalCDF(effL) is 0, i.e. when
    the fragment covers more than ~30 % of the transcript"""
    k = next(i for i in range(len(lines) - 2) if lines[i].strip() == "1" and lines[i + 1].strip() == "20"
             and len(lines[i + 2].split()) == 20)
    pdf = lines[k + 2].split()
    lines[k + 2] = " ".join(["0"] * 14 + pdf[14:])
    return lines


def test_failed_attempts_rspd(tmp_path):
    d = _case(tmp_path, "sim_rspd_fail", "pe_q_rspd", _zero_rspd_bins)
    out = _compare(d, "sim_rspd_fail", 0.1, 5000, 9)
    assert _resim(out) > 0
    d = _case(tmp_path, "sim_rspd_fail_win", "pe_q_rspd", _zero_rspd_bins)
    assert _resim(_compare(d, "sim_rspd_fail_win", 0.1, 20000, 13, env={"RSEM_B200_SIM_WINDOW": "2500"})) > 0


def _se_with_mld(lines):
    """single-end model with fragment lengths 20..200 and a mate-length distribution 30..40 (what
    --fragment-length-mean gives): reads of fragments shorter than 30 fail in SingleModel::simulate"""
    assert lines[0].strip() == "0" and lines[7].strip() == "0"
    gld = ["19 200 181", " ".join(["%.10g" % (1.0 / 181)] * 181)]
    mld = ["1", "29 40 11", " ".join(["%.10g" % (1.0 / 11)] * 11)]
    return lines[:4] + gld + lines[6:7] + mld + lines[8:]


def test_single_end_with_mld(tmp_path):
    d = _case(tmp_path, "sim_se_mld", "se_noq", _se_with_mld)
    assert _resim(_compare(d, "sim_se_mld", 0.1, 5000, 21)) > 0


def test_allele_specific_reference(tmp_path):
    """.gt / .ta next to the reference: TPM is read from column 7 (OFFSITE 6) and .sim.alleles.results is written"""
    d = _case(tmp_path, "sim_allele", "se_q_rspd", extra_col=True)
    grp = [int(x) for x in open(d / "ref" / "r.grp").read().split()]
    M = grp[-1] - 1
    # alleles 2k - 1 and 2k form transcript k where both lie in the same gene; otherwise an allele is its own transcript
    ta = [1]
    while ta[-1] <= M:
        a = ta[-1]
        ta.append(a + 2 if a + 1 <= M and not any(a < g <= a + 1 for g in grp) else a + 1)
    gt = [ta.index(g) for g in grp]
    open(d / "ref" / "r.ta", "w").write("\n".join(map(str, ta)) + "\n")
    open(d / "ref" / "r.gt", "w").write("\n".join(map(str, gt)) + "\n")
    _compare(d, "sim_allele", 0.2, 3000, 11)
    if not RECORD_ONLY:
        assert os.path.exists(str(d) + ".gpu/s.sim.alleles.results")


@pytest.mark.parametrize("final_newline", [True, False])
def test_results_file_with_too_few_lines(tmp_path, final_newline):
    """10 of M rows: after a final newline the missing rows read as TPM 0; without one, std::getline keeps the last
    row and every missing transcript repeats its TPM"""
    key = f"sim_short_{int(final_newline)}"
    d = _case(tmp_path, key, "se_noq", rows=10, final_newline=final_newline)
    _compare(d, key, 0.1, 3000, 11)


def test_zero_profile_rows(tmp_path):
    """the QProfile block of the most common quality set to 0: the reference leaves it unrepaired
    (QProfile.h:170), so simul::sample draws a second word for every base of that quality and the attempt lengths
    depend on the drawn qualities.  (A zero QualDist row cannot be used: its uniform fallback draws qualities above
    93, which the reference rejects with an assertion.)"""
    def edit(lines):
        k = next(i for i, l in enumerate(lines) if l.strip() == "100" and len(lines[i + 1].split()) == 100)  # QualDist
        init = [float(x) for x in lines[k + 1].split()]
        q = max(range(100), key=lambda i: init[i])
        k0 = next(i for i, l in enumerate(lines) if l.strip() == "100 5")  # QProfile: 100 blocks of 5 rows + a blank
        for r in range(5):
            lines[k0 + 1 + q * 6 + r] = " ".join(["0"] * 5)
        return lines
    d = _case(tmp_path, "sim_zero_rows", "pe_q_rspd", edit)
    _compare(d, "sim_zero_rows", 0.2, 4000, 17)
    d = _case(tmp_path, "sim_zero_rows_win", "pe_q_rspd", edit)
    _compare(d, "sim_zero_rows_win", 0.2, 20000, 4, env={"RSEM_B200_SIM_WINDOW": "5000"})
    d = _case(tmp_path, "sim_zero_rows_plain", "pe_q_rspd")
    _compare(d, "sim_zero_rows_plain", 0.2, 4000, 17)
    if not RECORD_ONLY:
        assert open(tmp_path / "sim_zero_rows.gpu" / "s_1.fq", "rb").read() != \
            open(tmp_path / "sim_zero_rows_plain.gpu" / "s_1.fq", "rb").read()


def test_seeds_differ(tmp_path):
    d = _case(tmp_path, "sim_seed1", "pe_noq")
    _compare(d, "sim_seed1", 0.2, 2000, 1)
    d2 = _case(tmp_path, "sim_seed2", "pe_noq")
    _compare(d2, "sim_seed2", 0.2, 2000, 2)
    if not RECORD_ONLY:
        assert open(str(d) + ".gpu/s_1.fa", "rb").read() != open(str(d2) + ".gpu/s_1.fa", "rb").read()
