"""Drop-in acceptance with --calc-ci: the UNMODIFIED Perl driver rsem-calculate-expression runs the whole pipeline with
--calc-ci --seed 42 -p 2 (rsem-parse-alignments, rsem-build-read-index, rsem-run-em, rsem-run-gibbs with the driver's
default 1000 count vectors, rsem-calculate-credibility-intervals with 50 samples per count vector) once with the
reference's binaries (oracle/_ref) and once with our four binaries swapped in beside the same driver.  The
*.isoforms.results and *.genes.results it writes from the appended rows, credibility intervals included, are compared
as the other acceptance tests compare them (0.011 absolute: the results print two decimals)."""
import os
import shutil
import subprocess

import pytest

import rsem_files as rf
from test_acceptance_gpu import DRIVER, _compare_tables

pytestmark = pytest.mark.gpu
TOOLS = ("rsem-parse-alignments", "rsem-run-em", "rsem-run-gibbs", "rsem-calculate-credibility-intervals")


def _install(dst, which):
    os.makedirs(dst)
    for f in ("rsem-calculate-expression", "rsem_perl_utils.pm"):
        shutil.copy(os.path.join(rf.REF_DIR, f), dst)
    os.symlink(os.path.join(rf.REF_DIR, "rsem-build-read-index"), os.path.join(dst, "rsem-build-read-index"))
    for tool in TOOLS:
        os.symlink(os.path.join(rf.REF_DIR if which == "ref" else rf.BIN_DIR, tool), os.path.join(dst, tool))
    return dst


def _run(bindir, work, data):
    os.makedirs(work)
    cmd = ["perl", os.path.join(bindir, "rsem-calculate-expression"), "--alignments", "--paired-end",
           "--keep-intermediate-files", "--calc-ci", "--seed", "42", "-p", "2", os.path.join(data, "aln.sam"),
           os.path.join(data, "ref", "r"), "smp"]
    p = subprocess.run(cmd, cwd=work, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-3000:]
    return p.stdout


def test_perl_driver_calc_ci(tmp_path, built):
    if not (os.path.exists(os.path.join(rf.REF_DIR, "rsem-calculate-credibility-intervals")) and os.path.exists(DRIVER)
            and shutil.which("perl")):
        pytest.skip("needs oracle/_ref with the Perl driver and the reference tool (oracle/Makefile, oracle/ci.mk) and perl")
    data = rf.gen_dataset(str(tmp_path / "data"), read_type=3, sam=1, seed=21, M=150, N1=3000, N0=150, read_len=50,
                          spurious=0.05)
    out_ref = _run(_install(str(tmp_path / "bin_ref"), "ref"), str(tmp_path / "ref"), data)
    out_ours = _run(_install(str(tmp_path / "bin_ours"), "ours"), str(tmp_path / "ours"), data)
    for out in (out_ref, out_ours):
        assert "rsem-calculate-credibility-intervals" in out and "All credibility intervals are calculated!" in out
    header = open(tmp_path / "ours" / "smp.isoforms.results").readline()
    assert "TPM_ci_lower_bound" in header and "FPKM_coefficient_of_quartile_variation" in header
    for f in ("smp.isoforms.results", "smp.genes.results"):
        _compare_tables(str(tmp_path / "ours" / f), str(tmp_path / "ref" / f))
