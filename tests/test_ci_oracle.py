"""The CPU restatement of Phase II (oracle/rsem_oracle.c: ro_ci_phase2) against the reference tool
(oracle/_ref/rsem-calculate-credibility-intervals, built by oracle/ci.mk; skipped where it is not built).

The reference runs on the pe_noq golden set's own count vectors and leaves its samples behind in imd.tmp (M rows of
nSamples float32, transcript-major).  The restatement takes that file and must print the TPM lb / ub / cqv rows the
reference appended to imd.iso_res (imd.allele_res) and imd.gene_res, with %.6g.  FPKM is not checked here: the
reference does not write its l_bars anywhere, and FPKM = 1e3 / l_bar * tpm needs them.  The bits of FPKM are held by
tests/test_ci_kernels_gpu.py, kernel against restatement."""
import os

import numpy as np
import pytest

import ci_phase2 as cp

pytestmark = pytest.mark.skipif(not os.path.exists(cp.REF_BIN), reason="oracle/_ref holds no reference tool")


def _check(oracle, run, l_bars):
    tr, ge, iso = oracle.ci_phase2(run["samples"], l_bars, run["gene_start"], run["threshold"],
                                   isoform_start=run["isoform_start"], part_gene_start=run["parts"])
    tr_file = "s.allele_res" if run["isoform_start"] else "s.iso_res"
    assert cp.text_rows(tr[:, :3]) == run["rows"][tr_file][:3]
    assert cp.text_rows(ge[:, :3]) == run["rows"]["s.gene_res"][:3]
    if run["isoform_start"]:
        assert cp.text_rows(iso[:, :3]) == run["rows"]["s.iso_res"][:3]
    return tr, ge, iso


@pytest.mark.parametrize("nspc", [50, 51])
def test_restatement_prints_the_reference_rows(oracle, tmp_path, nspc):
    """-p 2: two Phase II ranges; 300 and 306 samples (nSamples % 4 = 0 and 2)"""
    run = cp.reference_run(tmp_path, 2, nspc)
    assert len(run["parts"]) == 3
    _check(oracle, run, np.full(run["n"], 250.0, np.float32))


def test_restatement_allele_specific(oracle, tmp_path):
    """.ta / .gt with -p 1: the running isoform sums of the whole reference, sorted in place at each isoform with
    several alleles"""
    run = cp.reference_run(tmp_path, 1, 50, alleles=True)
    iso = run["isoform_start"]
    assert any(b - a > 1 for a, b in zip(iso, iso[1:])) and any(b - a == 1 for a, b in zip(iso, iso[1:]))
    _check(oracle, run, np.full(run["n"], 250.0, np.float32))
