"""bin/rsem-tbam2gbam against the reference's rsem-tbam2gbam (oracle/_ref, or its outputs stored under
tests/golden/reference/tbam2gbam_*): the same stdout, and the same genome BAM decoded field by field - header, every
record in order, tags in order with the exact ZW bits.  Inputs: genome-mode data sets (gene loci on both strands,
isoforms sharing a multi-exon body, so that a read's alignments collapse) plus hand-written records."""
import os
import random
import re
import subprocess

import pytest

import rsem_files as rf
import tbam2gbam as tg

pytestmark = pytest.mark.gpu


def _seq(rng, n):
    return "".join(rng.choice("ACGT") for _ in range(n))


def _hand_records(d, read_type, polyA):
    """records a generated data set lacks: poly(A) overlaps on both strands, MD and XS tags, mate 2 first, unmapped"""
    _, tr = tg.read_ti(os.path.join(d, "ref", "r.ti"))
    rng = random.Random(7)
    hasq, paired = read_type & 1, read_type >= 2
    picks = [next(i for i, t in enumerate(tr) if t[5] == s and t[6] >= 200) for s in "+-"]
    out = []

    def line(name, flag, t, pos, n, tags="", mpos=0, tlen=0):
        s = _seq(rng, n)
        q = "".join(chr(33 + rng.randrange(2, 41)) for _ in range(n)) if hasq else "*"
        rn = f"T{t + 1}" if t is not None else "*"
        cig = f"{n}M" if t is not None else "*"
        nxt = ("=" if t is not None else "*") if paired else "*"
        out.append("\t".join(str(x) for x in (name, flag, rn, pos, 255 if t is not None else 0, cig, nxt, mpos, tlen, s, q))
                   + ("\t" + tags if tags else ""))

    md = ["NM:i:3\tMD:Z:10A5^AC3T0G8\tXS:A:+\tXX:Z:keep", "MD:Z:7N2^GTa0C3\tNM:i:1", "XS:A:-\tMD:Z:3A^C2G", "MD:Z:0^T12"]
    for k, i in enumerate(picks):
        L = tr[i][6]
        if not paired:
            line(f"h{k}_tail_over", 0, i, L - 9, 30)
            line(f"h{k}_tail_in", 16, i, L + 3, min(15, polyA - 3))
            line(f"h{k}_start", 0, i, 1, 25, md[3])
            for j, tags in enumerate(md):
                line(f"h{k}_md{j}", 16 * (j & 1), i, 5 + j, 40, tags)
            line(f"h{k}_un", 4, None, 0, 30)
        else:
            line(f"h{k}_tail_over", 99, i, L - 9, 30, mpos=L + 2, tlen=31)
            line(f"h{k}_tail_over", 147, i, L + 2, 15, mpos=L - 9, tlen=-31)
            line(f"h{k}_m2first", 163, i, 40, 30, md[0], mpos=5, tlen=-65)   # mate 2 before mate 1
            line(f"h{k}_m2first", 83, i, 5, 30, md[1], mpos=40, tlen=65)
            line(f"h{k}_md", 99, i, 8, 40, md[2], mpos=60, tlen=92)
            line(f"h{k}_md", 147, i, 60, 40, md[3], mpos=8, tlen=-92)
            line(f"h{k}_un", 77, None, 0, 30)
            line(f"h{k}_un", 141, None, 0, 30)
    return out


def _case(tmp_path, read_type, hand=True, weight_step=0.0137, extra_lines=(), **kw):
    d = str(tmp_path / "d")
    polyA = kw.pop("polyA", 20)
    rf.gen_dataset(d, read_type=read_type, genome=1, sam=1, polyA=polyA, **kw)
    lines = open(os.path.join(d, "aln.sam")).read().splitlines()
    if hand:
        lines += _hand_records(d, read_type, polyA)
    lines += list(extra_lines)
    with open(os.path.join(d, "in.sam"), "w") as f:
        f.write("\n".join(lines) + "\n")
    tg.sam_to_bam(os.path.join(d, "in.sam"), os.path.join(d, "in.bam"), weight_step)
    os.remove(os.path.join(d, "in.sam"))
    return d


def _check(key, d, **kw):
    ref, ours, ref_digest, text = tg.run_pair(key, d, **kw)
    assert ref.returncode == 0, ref.stderr
    assert ours.returncode == 0, ours.stderr
    assert ours.stdout == ref.stdout
    if tg.os.path.exists(tg.REF_EXE):
        with open(d.rstrip("/") + "_ref/g.txt") as f:
            want = f.read()
        assert text == want, next((f"line {i}:\n ours {a}\n ref  {b}" for i, (a, b) in
                                   enumerate(zip(text.splitlines(), want.splitlines())) if a != b), "lengths differ")
    assert tg.sha(text) == ref_digest
    return text


CASES = {  # key: (read_type, gen_dataset arguments)
    "se_q": (1, dict(M=40, N1=400, N0=0, seed=3)),
    "se_noq": (0, dict(M=40, N1=400, N0=0, seed=4, var_len=10)),
    "pe_q": (3, dict(M=40, N1=300, N0=0, seed=5)),
    "pe_noq": (2, dict(M=40, N1=300, N0=0, seed=6)),
}


@pytest.mark.parametrize("key", sorted(CASES))
def test_matches_reference(built, tmp_path, key):
    read_type, kw = CASES[key]
    text = _check(key, _case(tmp_path, read_type, **kw))
    assert '"XS", "A", "-"' in text and '"XS", "A", "+"' in text   # spliced reads on both strands
    assert re.search(r'"cigar": "[0-9MIN]*N', text) and re.search(r'"cigar": "[0-9MIN]*I', text)   # introns, poly(A) overlaps


def test_without_zw(built, tmp_path):
    """an aligner's BAM: no ZW anywhere, so MAPQ 255 on every converted record and sums of 1.0 (never written)"""
    d = _case(tmp_path, 3, weight_step=0.0, M=30, N1=200, N0=0, seed=8)
    text = _check("no_zw", d)
    assert '"ZW"' not in text and '"mapq": 255' in text


def test_read_with_many_alignments(built, tmp_path):
    rng = random.Random(3)
    s = _seq(rng, 30)
    extra = [f"many\t0\tT{t}\t{p}\t255\t30M\t*\t0\t0\t{s}\t*" for t in range(1, 11) for p in range(1, 601)]
    d = _case(tmp_path, 0, hand=False, extra_lines=extra, M=30, N1=100, N0=0, seed=9, polyA=0)
    _check("many", d)
    # batches of a few dozen units first, then the 6000-unit group in one batch larger than the budget: the device
    # scratch must grow for it, and the file must not change
    w = tg._rundir(d, "small")
    p = subprocess.run([tg.OUR_EXE, "ref/r", "in.bam", "g.bam"], cwd=w, env=dict(os.environ, RSEM_B200_GBAM_BATCH="3000"),
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert p.returncode == 0, p.stderr
    assert open(os.path.join(w, "g.bam"), "rb").read() == open(d + "_ours/g.bam", "rb").read()


def test_small_batches_and_threads_give_identical_files(built, tmp_path):
    d = _case(tmp_path, 3, M=40, N1=300, N0=0, seed=5)
    _check("pe_q", d)
    base = open(d + "_ours/g.bam", "rb").read()
    for name, env, args in (("small", {"RSEM_B200_GBAM_BATCH": "3000"}, ()), ("p1", {}, ("-p", "1")),
                            ("p7", {"RSEM_B200_IO_THREADS": "7"}, ())):
        w = tg._rundir(d, name)
        e = dict(os.environ)
        e.update(env)
        p = subprocess.run([tg.OUR_EXE, "ref/r", "in.bam", "g.bam", *args], cwd=w, env=e, stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, text=True)
        assert p.returncode == 0, p.stderr
        other = open(os.path.join(w, "g.bam"), "rb").read()
        if args:   # the command line is in the header: compare the records
            assert tg.canonical(os.path.join(w, "g.bam")).split("\n", 1)[1] == tg.canonical(d + "_ours/g.bam").split("\n", 1)[1]
        else:
            assert other == base, name


def test_progress_dots(built, tmp_path):
    d = _case(tmp_path, 0, hand=False, M=600, N1=330000, N0=0, seed=12, avg_family=4, read_len=36)
    text = _check("dots", d)
    assert text.count("\n") > 300000


def test_rejects_a_partial_pair(built, tmp_path):
    bad = ["bad\t73\tT1\t5\t255\t30M\t=\t5\t0\t" + "A" * 30 + "\t*", "bad\t133\t*\t0\t0\t*\t*\t0\t0\t" + "C" * 30 + "\t*"]
    d = _case(tmp_path, 2, hand=False, extra_lines=bad, M=20, N1=50, N0=0, seed=13)
    ref, ours, _, _ = tg.run_pair("reject", d)
    assert ours.returncode == 255 and ref.returncode == 255
    assert ours.stdout == ref.stdout
    assert "Detected partial alignments for read bad, which RSEM currently does not support!" in ours.stderr
