"""Drop-in acceptance of bin/rsem-tbam2gbam: the UNMODIFIED Perl driver rsem-calculate-expression runs with
--output-genome-bam on a genome-mode data set, once with the reference's binaries (oracle/_ref) and once with ours,
bin/rsem-tbam2gbam included, beside the same driver.  The driver calls rsem-tbam2gbam without -p on the transcript BAM
rsem-run-em -b wrote (rsem-calculate-expression:649-653).  Compared: every record of *.genome.bam.  ZW comes from two
different EMs here, so ZW and MAPQ get test_acceptance_gpu.py's tolerance; every other field must be equal."""
import os
import shutil

import pytest

import rsem_files as rf
from bam_reader import read_bam
from test_acceptance_gpu import DRIVER, _install, _run

pytestmark = pytest.mark.gpu

CASES = {
    "pe_q": (3, ["--paired-end"], dict(M=60, N1=3000, N0=150, read_len=50, polyA=20)),
    "se_noq": (0, ["--no-qualities"], dict(M=60, N1=4000, N0=200, read_len=50)),
}


@pytest.fixture(scope="module")
def installs(tmp_path_factory, built):
    if not (rf.have_ref() and os.path.exists(DRIVER) and os.path.exists(os.path.join(rf.REF_DIR, "rsem-tbam2gbam"))
            and shutil.which("perl")):
        pytest.skip("needs oracle/_ref with the Perl driver and rsem-tbam2gbam (oracle/Makefile, oracle/tbam2gbam.mk) and perl")
    base = tmp_path_factory.mktemp("genome_bam")
    dirs = {}
    for which, src in (("ref", rf.REF_DIR), ("ours", rf.BIN_DIR)):
        d = _install(str(base / f"bin_{which}"), which)
        os.symlink(os.path.join(src, "rsem-tbam2gbam"), os.path.join(d, "rsem-tbam2gbam"))
        dirs[which] = d
    return base, dirs["ref"], dirs["ours"]


@pytest.mark.parametrize("name", list(CASES))
def test_perl_driver_output_genome_bam(installs, name):
    base, bin_ref, bin_ours = installs
    rt, flags, opts = CASES[name]
    data = rf.gen_dataset(str(base / f"{name}_data"), read_type=rt, sam=1, genome=1, seed=31, **opts)
    out_ref = _run(bin_ref, str(base / f"{name}_ref"), data, flags + ["--output-genome-bam"])
    out_ours = _run(bin_ours, str(base / f"{name}_ours"), data, flags + ["--output-genome-bam"])
    assert "rsem-tbam2gbam" in out_ref and "rsem-tbam2gbam" in out_ours
    wr, wo = str(base / f"{name}_ref"), str(base / f"{name}_ours")
    tr, rr, ref = read_bam(f"{wr}/smp.genome.bam")
    to, ro, ours = read_bam(f"{wo}/smp.genome.bam")
    # the @PG line holds each run's own command line (the same here: both drivers call it by name from PATH)
    assert (tr, rr) == (to, ro) and len(ref) == len(ours) > 0
    n_zw = n_spliced = 0
    for a, b in zip(ours, ref):
        za, zb = a["tags"].get("ZW"), b["tags"].get("ZW")
        assert (za is None) == (zb is None)
        if zb is not None:
            n_zw += 1
            assert za[0] == zb[0] == "f" and abs(za[1] - zb[1]) <= 1e-6 + 1e-6 * abs(zb[1]), (a, b)
            assert abs(a["mapq"] - b["mapq"]) <= (0 if za[1] == zb[1] else 1), (a, b)
            a["tags"]["ZW"], a["mapq"] = zb, b["mapq"]
        assert a == b
        n_spliced += "N" in a["cigar"]
    assert n_zw > 0 and n_spliced > 0
