"""CPU checks of bin/rsem-calculate-credibility-intervals' command line and the errors it reports before any device
work: the usage message, a missing count-vector file, count-vector files that do not hold nCV vectors, and the
reference's check that nMB holds one sample row (Buffer.h:18-20)."""
import os
import shutil
import subprocess
import tarfile

import pytest

import rsem_files as rf

BIN = os.path.join(rf.ROOT, "bin", "rsem-calculate-credibility-intervals")


def _run(*args, cwd=None):
    return subprocess.run([BIN, *args], capture_output=True, text=True, cwd=cwd)


@pytest.fixture
def imd(built, tmp_path):
    """the pe_noq golden set with the two count-vector files the reference's rsem-run-gibbs wrote (3 vectors each)"""
    with tarfile.open(os.path.join(rf.ROOT, "tests", "golden", "pe_noq.tar.gz")) as t:
        t.extractall(tmp_path, filter="data")
    d = tmp_path / "pe_noq"
    for i in range(2):
        shutil.copy(d / "out" / f"countvectors{i}", d / "s.temp" / f"s.countvectors{i}")
    shutil.copy(d / "out" / "model20", d / "s.stat" / "s.model")
    return d


def _args(ncv, nmb, *extra):
    return ["ref/r", "s.temp/s", "s.stat/s", "0.95", str(ncv), "10", str(nmb), *extra]


@pytest.mark.parametrize("n", [0, 3, 6])
def test_usage(built, n):
    p = _run(*(["x"] * n))
    assert p.returncode == 255
    assert p.stdout.startswith("Usage: rsem-calculate-credibility-intervals reference_name imdName statName confidence nCV nSpC nMB")


def test_missing_count_vector_file(imd):
    p = _run(*_args(9, 16, "-p", "3"), cwd=imd)
    assert p.returncode == 255
    assert "Cannot open s.temp/s.countvectors2! It may not exist." in p.stderr


@pytest.mark.parametrize("ncv", [5, 7])
def test_wrong_ncv(imd, ncv):
    p = _run(*_args(ncv, 16, "-p", "2"), cwd=imd)
    assert p.returncode == 255
    assert f"The count-vector files hold 6 count vectors, not nCV = {ncv}!" in p.stderr


def test_nmb_too_small(imd):
    p = _run(*_args(6, 0, "-p", "2"), cwd=imd)
    assert p.returncode == 255
    assert "Memory allocated for credibility intervals is not enough!" in p.stderr
    assert not os.path.exists(imd / "s.temp" / "s.tmp")
