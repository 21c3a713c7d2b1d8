"""CPU checks of bin/rsem-simulate-reads' command line: argument count, missing model file, and the error paths
that end before any device work."""
import os
import subprocess

import pytest

import rsem_files as rf

BIN = os.path.join(rf.ROOT, "bin", "rsem-simulate-reads")


def _run(*args):
    return subprocess.run([BIN, *args], capture_output=True, text=True)


@pytest.mark.parametrize("n", [0, 5, 10])
def test_wrong_argc_prints_usage(built, n):
    p = _run(*(["x"] * n))
    assert p.returncode == 255
    assert p.stdout.startswith("Usage: rsem-simulate-reads reference_name estimated_model_file")


def test_missing_model(built, tmp_path):
    ref = os.path.join(rf.ROOT, "dataset", "ref", "r")
    model = str(tmp_path / "none.model")
    p = _run(ref, model, str(tmp_path / "res"), "0.1", "10", str(tmp_path / "out"), "--seed", "1")
    assert p.returncode == 255
    assert f"Cannot open {model}! It may not exist." in p.stderr


def test_results_file_without_expression_aborts(built, tmp_path):
    """a results file with only its header line: every TPM reads as 0, and like the reference (simulation.cpp:113)
    the run aborts before any device work"""
    d = os.path.join(rf.ROOT, "tests", "golden", "se_noq.tar.gz")
    import tarfile
    with tarfile.open(d) as t:
        t.extractall(tmp_path, filter="data")
    res = tmp_path / "res.tsv"
    res.write_text("transcript_id\tgene_id\tlength\teffective_length\texpected_count\tTPM\tFPKM\tIsoPct\n")
    p = _run(str(tmp_path / "se_noq" / "ref" / "r"), str(tmp_path / "se_noq" / "out" / "model20"), str(res), "0.1", "10",
             str(tmp_path / "out"), "--seed", "1")
    assert p.returncode == -6
    assert os.path.exists(str(tmp_path / "out.fa"))  # the read file is created before the model is read
