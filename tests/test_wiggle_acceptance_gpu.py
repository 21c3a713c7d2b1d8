"""The reference's unmodified rsem-plot-transcript-wiggles with our rsem-bam2readdepth beside it: the read-depth file it
makes equals the reference tool's, and rsem-gen-transcript-plots (a stub here, the R step is out of scope) gets the
reference's arguments.  S.transcript.sorted.bam is placed beforehand, so no samtools is needed."""
import os
import shutil
import subprocess

import pytest

import rsem_files as rf
import tbam2gbam as tg
import wiggle as wg

pytestmark = pytest.mark.gpu

STUB = """#!/bin/sh
echo "$@" > gen_transcript_plots.args
"""


def test_plot_transcript_wiggles(built, tmp_path):
    script = os.path.join(rf.REF_DIR, "rsem-plot-transcript-wiggles")
    if not os.path.exists(script):
        pytest.skip("needs oracle/_ref")
    d = str(tmp_path / "d")
    rf.gen_dataset(d, read_type=3, M=40, N1=400, N0=0, seed=5, sam=1, polyA=0)
    tg.sam_to_bam(os.path.join(d, "aln.sam"), str(tmp_path / "raw.bam"), 0.0137)
    inst = str(tmp_path / "inst")
    os.makedirs(inst)
    for f in ("rsem-plot-transcript-wiggles", "rsem_perl_utils.pm"):
        shutil.copy(os.path.join(rf.REF_DIR, f), inst)
    os.symlink(wg.our_exe("depth"), os.path.join(inst, "rsem-bam2readdepth"))
    with open(os.path.join(inst, "rsem-gen-transcript-plots"), "w") as f:
        f.write(STUB)
    os.chmod(os.path.join(inst, "rsem-gen-transcript-plots"), 0o755)
    w = str(tmp_path / "w")
    os.makedirs(w)
    wg.sort_bam(str(tmp_path / "raw.bam"), os.path.join(w, "S.transcript.sorted.bam"))
    with open(os.path.join(w, "ids.txt"), "w") as f:
        f.write("T1\nT2\n")
    p = subprocess.run(["perl", os.path.join(inst, "rsem-plot-transcript-wiggles"), "S", "ids.txt", "out.pdf"], cwd=w,
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    r = subprocess.run([wg.ref_exe("depth"), "S.transcript.sorted.bam", "ref.readdepth"], cwd=w, stdout=subprocess.PIPE,
                       text=True)
    assert r.returncode == 0
    assert open(os.path.join(w, "S.transcript.readdepth"), "rb").read() == open(os.path.join(w, "ref.readdepth"), "rb").read()
    assert open(os.path.join(w, "gen_transcript_plots.args")).read() == "S ids.txt 0 1 0 out.pdf\n"
