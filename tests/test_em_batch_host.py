"""rsem-run-em-batch on the CPU: usage, the manifest refusals (all made before a GPU is touched or a file is written),
and the generator options that make samples sharing one reference."""
import filecmp
import os
import subprocess

import pytest

import rsem_files as rf

EXE = os.path.join(rf.BIN_DIR, "rsem-run-em-batch")


@pytest.fixture(scope="module")
def samples(built, tmp_path_factory):
    root = tmp_path_factory.mktemp("batch")
    return [rf.gen_dataset(str(root / f"d{k}"), read_type=0, M=60, N1=300, N0=10, sample_seed=k + 1) for k in range(3)]


def _run(cwd, manifest_text, read_type=0, extra=()):
    with open(os.path.join(cwd, "manifest"), "w") as f:
        f.write(manifest_text)
    ref = os.path.relpath(os.path.join(cwd, "d0", "ref", "r"), cwd)
    return subprocess.run([EXE, ref, str(read_type), "manifest", *extra], cwd=cwd, stdout=subprocess.PIPE,
                          stderr=subprocess.PIPE, text=True)


def _line(k, extra=""):
    return f"d{k}/s d{k}/s.temp/s d{k}/s.stat/s{extra}\n"


def _outputs(cwd):
    found = []
    for dirpath, _, files in os.walk(cwd):
        found += [f for f in files if f.endswith((".theta", ".model", ".iso_res", ".gene_res", ".ofg", ".transcript.bam"))]
    return found


def test_usage(built):
    p = subprocess.run([EXE], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert p.returncode == 255 and p.stdout.startswith("Usage")


@pytest.mark.parametrize("case", ["few_fields", "no_cnt", "bad_cnt", "read_type", "same_stat", "same_imd", "same_sample"])
def test_manifest_refusals(samples, case):
    cwd = os.path.dirname(samples[0])
    text = _line(0) + "\n"   # an empty line is skipped
    bad_no = 3
    if case == "few_fields":
        text += "d1/s d1/s.temp/s\n"
    elif case == "no_cnt":
        text += "d1/s d1/s.temp/s d1/s.stat/missing\n"
    elif case == "bad_cnt":
        with open(os.path.join(cwd, "d2", "s.stat", "garbled.cnt"), "w") as f:
            f.write("12 x\n")
        text += "d2/s d2/s.temp/s d2/s.stat/garbled\n"
    elif case == "read_type":
        text += _line(1)
    elif case == "same_stat":
        text += "d1/s d1/s.temp/s d0/s.stat/s\n"
    elif case == "same_imd":
        text += "d1/s d0/s.temp/s d1/s.stat/s\n"
    else:
        text += "d0/s d1/s.temp/s d1/s.stat/s\n"
    p = _run(cwd, text, read_type=1 if case == "read_type" else 0)
    if case == "read_type":
        bad_no = 1   # every line has read type 0: the first one is refused
    assert p.returncode == 255, p.stderr
    assert f"manifest line {bad_no}:" in p.stderr
    assert p.stdout == ""
    assert _outputs(cwd) == []


def test_sample_seed_shares_the_reference(samples):
    a, b = samples[0], samples[1]
    cmp = filecmp.dircmp(os.path.join(a, "ref"), os.path.join(b, "ref"))
    assert cmp.left_list == cmp.right_list and not cmp.diff_files and not cmp.funny_files
    for f in cmp.common_files:
        assert filecmp.cmp(os.path.join(a, "ref", f), os.path.join(b, "ref", f), shallow=False)
    assert not filecmp.cmp(os.path.join(a, "s.temp", "s.dat"), os.path.join(b, "s.temp", "s.dat"), shallow=False)
    assert not filecmp.cmp(rf.read_files(a, 0)[0], rf.read_files(b, 0)[0], shallow=False)


def test_expressed_frac_narrows_the_transcripts_hit(built, tmp_path):
    full = rf.gen_dataset(str(tmp_path / "full"), read_type=0, M=400, N1=3000, N0=10)
    few = rf.gen_dataset(str(tmp_path / "few"), read_type=0, M=400, N1=3000, N0=10, expressed_frac=0.1)

    def hit_set(d):
        _, sid = rf.read_dat(os.path.join(d, "s.temp", "s.dat"), False)[:2]
        return {abs(int(x)) for x in sid}

    assert len(hit_set(few)) < len(hit_set(full)) / 3
