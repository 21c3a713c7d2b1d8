"""rsem-bam2wig and rsem-bam2readdepth without a GPU: every usage and argument error, a missing input, an unwritable
output, header-only and all-unmapped inputs (none of which may create a CUDA context), and the two writers' formatting
against Python's %.2f / %.6g through the host self-test, in chunks down to one position."""
import math
import os
import struct
import subprocess

import pytest

import wiggle as wg

REFS = [("chrA", 40), ("tr2", 7), ("zero", 0), ("chrB", 1000)]
NO_GPU = {"CUDA_VISIBLE_DEVICES": ""}   # a CUDA context cannot be created: the run must not need one


def _usage_args():
    return {"wig": [[], ["a"], ["a", "b"], ["a", "b", "c", "d", "e"], ["a", "b", "c", "--bad"], ["a", "b", "c", "-p"]],
            "depth": [[], ["a"], ["a", "b", "c"], ["a", "b", "c", "d"]]}


@pytest.mark.parametrize("tool", ["wig", "depth"])
def test_usage_and_argument_errors(built, tmp_path, tool):
    for i, a in enumerate(_usage_args()[tool]):
        d = str(tmp_path / f"u{i}")
        os.makedirs(d)

        def run():
            return subprocess.run([wg.ref_exe(tool), *a], cwd=d, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        ref = wg.rf.reference_run(f"wiggle_usage_{tool}_{i}", d, run, digests_only=True)
        ours = subprocess.run([wg.our_exe(tool), *a], cwd=d, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        assert ours.returncode == ref.returncode == 255
        assert ours.stdout == ref.stdout and ours.stderr == ref.stderr


@pytest.mark.parametrize("tool", ["wig", "depth"])
def test_missing_input(built, tmp_path, tool):
    d = str(tmp_path / "d")
    os.makedirs(d)
    ref, ours = wg.run_pair(f"missing_{tool}", d, tool, infile="no_such.bam", env=NO_GPU)
    assert ours.returncode == ref.returncode == 255
    assert ours.stdout == ref.stdout and ours.stderr == ref.stderr
    assert wg.sha(ours.output) == ref.digests[wg.OUT[tool]]
    if tool == "wig":   # the track line is out before the input is opened
        assert ours.output == b'track type=wiggle_0 name="trk" description="trk" visibility=full\n'


def test_unwritable_output(built, tmp_path):
    d = str(tmp_path / "d")
    os.makedirs(d)
    wg.write_bam(os.path.join(d, "in.bam"), REFS, [])

    def run():
        return subprocess.run([wg.ref_exe("depth"), "in.bam", "no/such/dir/x"], cwd=d, stdout=subprocess.PIPE,
                              stderr=subprocess.PIPE, text=True)
    ref = wg.rf.reference_run("wiggle_unwritable_depth", d, run, digests_only=True)
    ours = subprocess.run([wg.our_exe("depth"), "in.bam", "no/such/dir/x"], cwd=d, stdout=subprocess.PIPE,
                          stderr=subprocess.PIPE, text=True)
    assert ours.returncode == ref.returncode == 255 and ours.stdout == ref.stdout and ours.stderr == ref.stderr
    # the reference's rsem-bam2wig crashes in fprintf(NULL) here; ours refuses
    p = subprocess.run([wg.our_exe("wig"), "in.bam", "no/such/dir/x", "t"], cwd=d, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True)
    assert p.returncode == 255 and "cannot open no/such/dir/x for writing" in p.stderr


@pytest.mark.parametrize("tool", ["wig", "depth"])
@pytest.mark.parametrize("case", ["header_only", "all_unmapped"])
def test_no_mapped_records(built, tmp_path, tool, case):
    d = str(tmp_path / "d")
    os.makedirs(d)
    recs = [] if case == "header_only" else [
        wg.record(f"u{i}", 4, -1 if i % 2 else i % 3, 5 if i % 2 == 0 else -1, [(20, wg.M)], wg.zwf(0.5)) for i in range(50)]
    wg.write_bam(os.path.join(d, "in.bam"), REFS, recs)
    ref, ours = wg.check_same(f"{case}_{tool}", d, tool, env=NO_GPU)
    assert ours.returncode == 0, ours.stderr
    if tool == "depth":
        assert ours.output.decode() == "".join(f"{n}\t{l}\tNA\n" for n, l in REFS)
    else:
        assert ours.output == b'track type=wiggle_0 name="trk" description="trk" visibility=full\n'


@pytest.mark.parametrize("tool", ["wig", "depth"])
@pytest.mark.parametrize("case", ["text", "refs"])
def test_truncated_bam_header(built, tmp_path, tool, case):
    """a BAM header cut short: htslib's message and the reference's `Cannot load SAM header!`, status 255"""
    d = str(tmp_path / "d")
    os.makedirs(d)
    if case == "text":   # l_text says 100, 11 bytes follow
        raw = b"BAM\1" + struct.pack("<i", 100) + b"@HD\tVN:1.4\n"
    else:                # two targets announced, one present
        raw = b"BAM\1" + struct.pack("<ii", 0, 2) + struct.pack("<i", 3) + b"ab\0"
    with open(os.path.join(d, "in.bam"), "wb") as f:
        f.write(wg.tg.bgzf(raw))
    ref, ours = wg.run_pair(f"truncated_header_{case}_{tool}", d, tool, env=NO_GPU)
    assert ours.returncode == ref.returncode == 255
    assert ours.stdout == ref.stdout and ours.stderr == ref.stderr
    assert "Cannot load SAM header!" in ours.stderr
    assert wg.sha(ours.output) == ref.digests[wg.OUT[tool]]


# ---- the writers' formatting -------------------------------------------------------------------------------------------
def _c_g(x):
    """glibc's %.6g (Python's %g drops a NaN's sign)"""
    if math.isnan(x):
        return "-nan" if math.copysign(1.0, x) < 0 else "nan"
    return "%.6g" % x


def _expect(values, lengths, wig):
    out, at = [], 0
    for k, L in enumerate(lengths):
        name = f"t{k}"
        empty = isinstance(L, str)
        n = int(L[1:]) if empty else L
        v = [] if empty or n == 0 else values[at:at + n]
        at += 0 if empty else n
        if wig:
            prev = False
            for i, x in enumerate(v):
                on = x >= 0.0095
                if on and not prev:
                    out.append(f"fixedStep chrom={name} start={i + 1} step=1\n")
                if on:
                    out.append("%.2f\n" % x)
                prev = on
        else:
            out.append(f"{name}\t{n}\t" + ("NA" if not v else " ".join(_c_g(x) for x in v)) + "\n")
    return "".join(out)


VALUES = [0.0, 0.125, 0.375, 2.675, 0.0095, 0.009499999999999999, 0.009500000000000001, 1e-5, 1.5e-7, 123456.5,
          1234567.0, 0.0001, 1e300, -2.5, -0.0, float("inf"), float("-inf"), float("nan"), -float("nan"),
          0.01, 0.02, 0.0, 0.015, 0.005, 0.0096, 5e-324, 99999.95, 0.999995, 1.0, 3.0, 1.7976931348623157e308]


@pytest.mark.parametrize("wig", [True, False])
def test_formatting_against_python(built, tmp_path, wig):
    vals = VALUES * 3 + [0.011 * i for i in range(40)]
    lengths = [len(VALUES), "e5", 0, len(VALUES) * 2, 1, "e0", 39]
    path = str(tmp_path / "v.f64")
    with open(path, "wb") as f:
        f.write(struct.pack(f"<{len(vals)}d", *vals))
    want = _expect(vals, lengths, wig)
    assert "fixedStep" in want or not wig
    for chunk, threads in ((1, 1), (1, 4), (3, 3), (7, 2), (1 << 16, 8)):
        out = str(tmp_path / f"o_{chunk}_{threads}")
        subprocess.run([wg.SELFTEST, "--wig-format", "wig" if wig else "depth", str(chunk), str(threads), path, out,
                        *[str(x) for x in lengths]], check=True, stdout=subprocess.DEVNULL)
        got = open(out).read()
        assert got == want, (chunk, threads, next((i for i, (a, b) in enumerate(zip(got, want)) if a != b), None))
    if wig:
        assert "\n0.12\n" in want and "\n0.38\n" in want
    else:
        assert " 0.125 " in want and " -nan " in want and " nan " in want and " inf " in want and " 1e-05 " in want
