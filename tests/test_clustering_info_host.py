"""CPU checks of bin/rsem-for-ebseq-calculate-clustering-info: the usage message, a missing input, and the cases that
need no device work (no transcripts, every transcript shorter than k, k <= 0), byte for byte against the reference tool
(oracle/_ref, or its stored runs under tests/golden/reference/ebseq_*.tar.xz).  Also checks the sort-based C restatement
(oracle/libkmer_oracle.so), with a Python reading of the FASTA, against the reference's stored outputs of every case the
GPU tests run."""
import hashlib
import os
import subprocess

import pytest

import clustering_info as ci


@pytest.mark.parametrize("n", [0, 1, 2, 4])
def test_usage(built, n):
    p = subprocess.run([ci.BIN, *(["1"] * n)], capture_output=True, text=True)
    assert p.returncode == 255
    assert p.stdout == f"Usage: {ci.TOOL} k input_reference_fasta_file output_file\n"


def test_missing_input(built, tmp_path):
    p = subprocess.run([ci.BIN, "25", "missing.fa", "out"], cwd=tmp_path, capture_output=True, text=True)
    assert p.returncode == 255
    assert "Cannot open missing.fa! It may not exist." in p.stderr
    assert not os.path.exists(tmp_path / "out")


@pytest.mark.parametrize("key", sorted(ci.HOST_CASES))
def test_no_device_work(built, tmp_path, key):
    """these cases must not need a device: they run on machines without one"""
    k, make = ci.HOST_CASES[key]
    ref = ci.write_case(str(tmp_path / "ref"), make())
    ours = ci.write_case(str(tmp_path / "ours"), make())
    r = ci.reference(key, ref, k)
    p = ci.run(ci.BIN, ours, k)
    assert r.returncode == 0 and p.returncode == 0, p.stderr
    assert p.stdout == r.stdout
    assert hashlib.sha256(open(os.path.join(ours, ci.OUT), "rb").read()).hexdigest() == r.digests[ci.OUT]


@pytest.mark.parametrize("key", sorted({**ci.DEVICE_CASES, **ci.HOST_CASES}))
def test_restatement_matches_reference(built, tmp_path, key):
    k, make = {**ci.DEVICE_CASES, **ci.HOST_CASES}[key]
    data = make()
    r = ci.reference(key, ci.write_case(str(tmp_path), data), k)
    kk = ci.atoi(k)
    names, off, bases, warnings = ci.load_ref(data)
    counts = ci.oracle_counts(kk, off, bases)
    text = ci.output_text(names, counts, ci.eff_lengths(kk, off))
    assert ci.stdout_text(kk, warnings) == r.stdout
    assert hashlib.sha256(text).hexdigest() == r.digests[ci.OUT]
