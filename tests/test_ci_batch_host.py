"""rsem-calculate-credibility-intervals-batch on the CPU: usage, an empty manifest and the manifest refusals, all made
before a CUDA context is created or a result file is touched (none of them needs a GPU).  Inputs: the pe_noq golden set
with the two count-vector files the reference's rsem-run-gibbs wrote (3 vectors each), as in test_ci_host.py."""
import hashlib
import os
import shutil
import subprocess
import tarfile

import pytest

import rsem_files as rf

EXE = os.path.join(rf.BIN_DIR, "rsem-calculate-credibility-intervals-batch")


@pytest.fixture(scope="module")
def root(built, tmp_path_factory):
    root = tmp_path_factory.mktemp("cibatch")
    with tarfile.open(os.path.join(rf.ROOT, "tests", "golden", "pe_noq.tar.gz")) as t:
        t.extractall(root, filter="data")
    d = root / "pe_noq"
    for i in range(2):
        shutil.copy(d / "out" / f"countvectors{i}", d / "s.temp" / f"s.countvectors{i}")
    shutil.copy(d / "out" / "model20", d / "s.stat" / "s.model")
    for f in ("iso_res", "gene_res"):   # result files the rows would be appended to
        shutil.copy(d / "out" / f"{f}_gibbs", d / "s.temp" / f"s.{f}")
    M = int(open(d / "ref" / "r.ti").readline().split()[0])
    lines = open(d / "out" / "model20").read().split("\n")
    k = max(i for i, x in enumerate(lines) if x.strip() == str(M))   # the mw block's header: M
    wide = list(lines)
    wide[k] = str(M + 1)
    open(d / "s.stat" / "wide.model", "w").write("\n".join(wide))
    open(d / "s.stat" / "cut.model", "w").write("\n".join(lines[:3]))
    os.makedirs(d / "t.temp")
    shutil.copy(d / "out" / "countvectors0", d / "t.temp" / "t.countvectors0")
    return d


def _run(d, text, *extra):
    with open(d / "manifest", "w") as f:
        f.write(text)
    return subprocess.run([EXE, "ref/r", "manifest", *extra], cwd=d, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                          text=True)


def _results(d):
    """digest of every result file under d"""
    out = {}
    for dp, _, fs in os.walk(d):
        for f in fs:
            if f.endswith(("iso_res", "gene_res", "allele_res")):
                out[os.path.join(dp, f)] = hashlib.sha256(open(os.path.join(dp, f), "rb").read()).hexdigest()
    return out


def test_usage(built):
    p = subprocess.run([EXE], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert p.returncode == 255
    assert p.stdout.startswith("Usage: rsem-calculate-credibility-intervals-batch reference_name manifest [-q]")


def test_empty_manifest(root):
    before = _results(root)
    p = _run(root, "\n  \n")
    assert p.returncode == 0, p.stderr
    assert p.stdout == "" and p.stderr == ""
    assert _results(root) == before


GOOD = "s.temp/s s.stat/s 0.95 6 10 16 -p 2 --seed 1"
CASES = {
    "few_fields": ("s.temp/s s.stat/s 0.95 6 10", "expected at least 6 fields"),
    "ncv_zero": ("t.temp/t s.stat/s 0.95 0 10 16 --seed 1", "nCV and nSpC must be positive!"),
    "nspc_negative": ("t.temp/t s.stat/s 0.95 3 -1 16 --seed 1", "nCV and nSpC must be positive!"),
    "too_many_samples": ("t.temp/t s.stat/s 0.95 3 715827883 16 --seed 1", "nCV * nSpC must be below 2^31!"),
    "nmb": ("t.temp/t s.stat/s 0.95 3 10 0 --seed 1", "Memory allocated for credibility intervals is not enough!"),
    "threads": ("t.temp/t s.stat/s 0.95 3 10 16 -p 0 --seed 1", "Number of threads should be bigger than 0!"),
    "seed_value": ("t.temp/t s.stat/s 0.95 3 10 16 --seed 12x", "cannot parse seed 12x"),
    "seed_missing": ("t.temp/t s.stat/s 0.95 3 10 16 -p 1 --seed", "--seed needs a value"),
    "no_model": ("t.temp/t s.stat/missing 0.95 3 10 16 --seed 1", "Cannot open s.stat/missing.model! It may not exist."),
    "model_cut": ("t.temp/t s.stat/cut 0.95 3 10 16 --seed 1", "Cannot parse a length distribution in the .model file!"),
    "model_M": ("t.temp/t s.stat/wide 0.95 3 10 16 --seed 1", "does not carry mask weights for this reference"),
    "no_count_vectors": ("t.temp/t s.stat/s 0.95 3 10 16 -p 2 --seed 1", "cannot open t.temp/t.countvectors1"),
    "same_imd": ("s.temp/../s.temp/s s.stat/s 0.5 6 10 16 -p 2 --seed 2", "imdName s.temp/../s.temp/s is line 1's too"),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_manifest_refusals(root, case):
    # an empty line is skipped and counted: the bad line is line 3
    line, why = CASES[case]
    before = _results(root)
    p = _run(root, GOOD + "\n\n" + line + "\n")
    assert p.returncode == 255, p.stderr
    assert "manifest line 3: " in p.stderr and why in p.stderr, p.stderr
    assert "ctx_create" not in p.stderr
    assert p.stdout == ""
    assert _results(root) == before
