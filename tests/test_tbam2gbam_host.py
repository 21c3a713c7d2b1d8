"""rsem-tbam2gbam without a GPU: the usage message, the refusal of a reference without genome information, the .ti
parse, the rewritten header (a header-only input needs no device) and the MAPQ threshold table the device uses."""
import os
import subprocess

import pytest

import rsem_files as rf
import tbam2gbam as tg

HEADERS = {
    "hdr_mixed": "@HD\tVN:1.4\tSO:unsorted\n@SQ\tSN:x\tLN:5\n@RG\tID:g1\n@PG\tID:RSEM\tCL:rsem-run-em a b\n"
                 "@PG\tID:bowtie2\tPN:bowtie2\tVN:2.2\n@CO\tone comment\n@CO\tanother\n@XY\tother line\n",
    "hdr_pg_only_field": "@HD\tVN:1.4\n@PG\tID:rsem-tbam2gbam\n@PG\tID:RSEM\n",
    "hdr_pg_with_cl": "@HD\tVN:1.4\n@PG\tID:rsem-tbam2gbam\tCL:rsem-tbam2gbam r in.bam out.bam\n@CO\tc\n",
    "hdr_empty": "",
}


def _genome_set(d, **kw):
    rf.gen_dataset(d, M=12, N1=20, N0=0, genome=1, **kw)
    return d


def _refs(d):
    _, tr = tg.read_ti(os.path.join(d, "ref", "r.ti"))
    return [(t[0], t[6]) for t in tr]


def test_usage(built):
    for args in ([], ["a"], ["a", "b", "c", "d"]):
        p = subprocess.run([tg.OUR_EXE, *args], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        assert p.returncode == 255
        assert p.stdout == ("Usage: rsem-tbam2gbam reference_name unsorted_transcript_bam_input genome_bam_output "
                            "[-p number_of_threads]\n")


def test_ti_type0_parse(built, tmp_path):
    d = _genome_set(str(tmp_path / "d"), polyA=20)
    typ, tr = tg.read_ti(os.path.join(d, "ref", "r.ti"))
    out = subprocess.run([tg.SELFTEST, "--ti", os.path.join(d, "ref", "r.ti")], stdout=subprocess.PIPE, text=True,
                         check=True).stdout.split("\n")
    assert out[0] == f"{len(tr)} {typ}" and typ == 0
    strands = set()
    for line, t in zip(out[1:], tr):
        f = line.split("\t")
        exons = [tuple(int(x) for x in e.split("-")) for e in f[8:]]
        assert f[:6] == [t[0], t[1], t[2], t[3], t[4], t[5]] and int(f[6]) == t[6] and exons == t[7]
        assert int(f[7]) == sum(e - s + 1 for s, e in t[7]) == t[6]
        strands.add(t[5])
    assert strands == {"+", "-"}


def test_refuses_reference_without_genome(built, tmp_path):
    d = rf.gen_dataset(str(tmp_path / "d"), M=12, N1=20, N0=0)   # .ti type 1
    tg.header_only_bam(os.path.join(d, "in.bam"), "@HD\tVN:1.4\n", _refs(d))
    ref, ours, _, _ = tg.run_pair("type1", d)
    assert ours.returncode == ref.returncode == 255
    assert ours.stdout == ref.stdout == "Start converting:\n"
    assert "Genome information is not provided! RSEM cannot convert the transcript bam file!" in ours.stderr
    assert ref.stderr.strip() in ours.stderr


@pytest.mark.parametrize("key", sorted(HEADERS))
def test_header_matches_reference(built, tmp_path, key):
    d = _genome_set(str(tmp_path / "d"))
    tg.header_only_bam(os.path.join(d, "in.bam"), HEADERS[key], _refs(d))
    ref, ours, ref_digest, text = tg.run_pair(key, d)
    assert ref.returncode == 0 and ours.returncode == 0, ours.stderr
    assert ours.stdout == ref.stdout == "Start converting:\nGenome bam file is generated!\n"
    assert tg.sha(text) == ref_digest, text
    if key == "hdr_pg_only_field":
        assert "@PG\\tID:rsem-tbam2gbam\\tCL:" not in text and text.count("@PG\\tID:rsem-tbam2gbam") == 1
    if key == "hdr_pg_with_cl":
        assert text.count("@PG\\tID:rsem-tbam2gbam") == 2


def test_mapq_table_every_float_in_0_2(built):
    """the device's MAPQ is #{m : prb >= t[m]}; checked against bam_prb_to_mapq (the host's log10) for all 2^30 + 1
    floats in [0, 2], which also shows the formula does not decrease there"""
    p = subprocess.run([tg.SELFTEST, "--mapq-table"], stdout=subprocess.PIPE, text=True)
    assert p.returncode == 0 and p.stdout == "1073741825 floats, 0 mismatches\n", p.stdout
