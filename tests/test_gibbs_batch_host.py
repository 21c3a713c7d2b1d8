"""rsem-run-gibbs-batch on the CPU: usage and the manifest refusals, all made before a CUDA context is created or a file
is written (this machine needs no GPU for them)."""
import os
import subprocess

import pytest

import rsem_files as rf

EXE = os.path.join(rf.BIN_DIR, "rsem-run-gibbs-batch")
M = 60


@pytest.fixture(scope="module")
def root(built, tmp_path_factory):
    """three samples of one reference with the files rsem-run-gibbs reads: .ofg, .omit, .model"""
    root = tmp_path_factory.mktemp("gbatch")
    for k in range(3):
        d = rf.gen_dataset(str(root / f"d{k}"), read_type=0, M=M, N1=50, N0=10, sample_seed=k + 1)
        with open(os.path.join(d, "s.temp", "s.ofg"), "w") as f:
            f.write(f"{M} 10\n" + "".join(f"0 0.5 {1 + i % M} 0.5\n" for i in range(50)))
        os.makedirs(os.path.join(d, "s.stat"), exist_ok=True)
        with open(os.path.join(d, "s.stat", "s.model"), "w") as f:
            f.write("0\n0.5\n")
    with open(root / "prior.txt", "w") as f:
        f.write("".join(f"{0.1 + i % 3} a comment\n" for i in range(M)))
    with open(root / "short_prior.txt", "w") as f:
        f.write("".join("1.0\n" for _ in range(M - 1)))
    return str(root)


def _line(k, rest="4 6 1 -p 2 --seed 3"):
    return f"d{k}/s.temp/s d{k}/s.stat/s {rest}\n"


def _outputs(cwd):
    found = []
    for _, _, files in os.walk(cwd):
        found += [f for f in files if ".countvectors" in f or f.endswith((".iso_res", ".gene_res"))]
    return found


def test_usage(built):
    p = subprocess.run([EXE], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert p.returncode == 255 and p.stdout.startswith("Usage: rsem-run-gibbs-batch refName manifest")


CASES = ["few_fields", "nsamples", "gap", "no_ofg", "bad_ofg", "ofg_M", "no_omit", "bad_omit", "no_model", "bad_model",
         "no_prior", "short_prior", "same_imd"]


@pytest.mark.parametrize("case", CASES)
def test_manifest_refusals(root, case):
    bad = {
        "few_fields": "d1/s.temp/s d1/s.stat/s 4 6\n",
        "nsamples": _line(1, "4 1 1"),
        "gap": _line(1, "4 6 0"),
        "no_ofg": "d1/s.temp/missing d1/s.stat/s 4 6 1\n",
        "bad_ofg": "d2/s.temp/garbled d2/s.stat/s 4 6 1\n",
        "ofg_M": "d2/s.temp/wide d2/s.stat/s 4 6 1\n",
        "no_omit": "d2/s.temp/noomit d2/s.stat/s 4 6 1\n",
        "bad_omit": "d2/s.temp/badomit d2/s.stat/s 4 6 1\n",
        "no_model": "d1/s.temp/s d1/s.stat/missing 4 6 1\n",
        "bad_model": "d1/s.temp/s d1/s.stat/garbled 4 6 1\n",
        "no_prior": _line(1, "4 6 1 --prior missing_prior.txt"),
        "short_prior": _line(1, "4 6 1 --prior short_prior.txt"),
        "same_imd": "d0/s.temp/s d1/s.stat/s 4 6 1\n",
    }[case]
    t = os.path.join(root, "d2", "s.temp")
    with open(os.path.join(t, "garbled.ofg"), "w") as f:
        f.write("x y\n")
    for name, text in (("wide", f"{M + 1} 0\n"), ("noomit", f"{M} 0\n"), ("badomit", f"{M} 0\n")):
        with open(os.path.join(t, name + ".ofg"), "w") as f:
            f.write(text)
    for name in ("wide", "badomit"):
        with open(os.path.join(t, name + ".omit"), "w") as f:
            f.write(f"3 {M + 1}\n" if name == "badomit" else "")
    with open(os.path.join(root, "d1", "s.stat", "garbled.model"), "w") as f:
        f.write("seven\n")
    with open(os.path.join(root, "manifest"), "w") as f:
        f.write(_line(0) + "\n" + bad)   # an empty line is skipped: the bad line is line 3
    p = subprocess.run([EXE, "d0/ref/r", "manifest"], cwd=root, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert p.returncode == 255, p.stderr
    assert "manifest line 3:" in p.stderr, p.stderr
    assert "ctx_create" not in p.stderr
    assert p.stdout == ""
    assert _outputs(root) == []
