"""rsem-simulate-reads-batch on the CPU: usage, an empty manifest and the manifest refusals, all made before a CUDA
context is created or a file is written (none of them needs a GPU)."""
import os
import subprocess
import tarfile

import pytest

import rsem_files as rf

EXE = os.path.join(rf.BIN_DIR, "rsem-simulate-reads-batch")


@pytest.fixture(scope="module")
def root(built, tmp_path_factory):
    """the se_noq golden reference and model, a results file, and models edited for the refusals"""
    root = tmp_path_factory.mktemp("simbatch")
    with tarfile.open(os.path.join(rf.ROOT, "tests", "golden", "se_noq.tar.gz")) as t:
        t.extractall(root, filter="data")
    d = root / "se_noq"
    M = int(open(d / "ref" / "r.ti").readline().split()[0])
    lines = open(d / "out" / "model20").read().split("\n")
    open(root / "model", "w").write("\n".join(lines))
    k = max(i for i, x in enumerate(lines) if x.strip() == str(M))   # the mw block's header: M
    wide = list(lines)
    wide[k] = str(M + 1)
    open(root / "wide.model", "w").write("\n".join(wide))
    open(root / "type7.model", "w").write("7\n" + "\n".join(lines[1:]))
    open(root / "cut.model", "w").write("\n".join(lines[:3]))
    rows = ["transcript_id\tgene_id\tlength\teffective_length\texpected_count\tTPM\tFPKM\tIsoPct"]
    rows += [f"T{i}\tG\t1\t1\t1\t{1 + i % 5}.00\t0\t0" for i in range(1, M + 1)]
    open(root / "res.tsv", "w").write("\n".join(rows) + "\n")
    os.makedirs(root / "sub")
    return str(root)


def _run(root, text, *extra):
    with open(os.path.join(root, "manifest"), "w") as f:
        f.write(text)
    return subprocess.run([EXE, "se_noq/ref/r", "manifest", *extra], cwd=root, stdout=subprocess.PIPE,
                          stderr=subprocess.PIPE, text=True)


def _outputs(root):
    """the read files and results tables outside the golden data set"""
    found = []
    for d, _, files in os.walk(root):
        if not os.path.relpath(d, root).startswith("se_noq"):
            found += [f for f in files if f.endswith((".fa", ".fq", ".results"))]
    return found


def test_usage(built):
    p = subprocess.run([EXE], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert p.returncode == 255
    assert p.stdout.startswith("Usage: rsem-simulate-reads-batch reference_name manifest [-q]")


def test_empty_manifest(root):
    p = _run(root, "\n  \n")
    assert p.returncode == 0, p.stderr
    assert p.stdout == "" and p.stderr == ""
    assert _outputs(root) == []


CASES = {
    "few_fields": "model res.tsv 0.1 100\n",
    "many_fields": "model res.tsv 0.1 100 b --seed 1 -q -q\n",
    "seed_value": "model res.tsv 0.1 100 b --seed x\n",
    "seed_missing": "model res.tsv 0.1 100 b -q --seed\n",
    "no_model": "missing.model res.tsv 0.1 100 b --seed 1\n",
    "model_type": "type7.model res.tsv 0.1 100 b --seed 1\n",
    "model_cut": "cut.model res.tsv 0.1 100 b --seed 1\n",
    "model_M": "wide.model res.tsv 0.1 100 b --seed 1\n",
    "no_results": "model missing.tsv 0.1 100 b --seed 1\n",
    "same_output": "model res.tsv 0.2 50 a --seed 2\n",
    "same_output_path": "model res.tsv 0.2 50 sub/../a --seed 2\n",
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_manifest_refusals(root, case):
    # an empty line is skipped and counted: the bad line is line 3
    p = _run(root, "model res.tsv 0.1 100 a --seed 1\n\n" + CASES[case])
    assert p.returncode == 255, p.stderr
    assert "manifest line 3:" in p.stderr, p.stderr
    assert "ctx_create" not in p.stderr
    assert p.stdout == ""
    assert _outputs(root) == []
