"""bin/rsem-bam2wig and bin/rsem-bam2readdepth against the reference's tools (oracle/_ref, or their outputs stored
under tests/golden/reference/wiggle_*): the same stdout, exit status and output file, byte for byte.  Inputs: sorted
transcript BAMs from generated data sets, a sorted genome BAM from rsem-tbam2gbam, hand-written records (every CIGAR
operation, ZW of every type, non-finite weights, a target that comes back), 1.2 M records for the progress lines, and
forced batching.  Then the refusals, and K11's sums against a NumPy restatement bit for bit."""
import os
import random
import struct
import subprocess

import numpy as np
import pytest

import bam_reader
import rsem_files as rf
import tbam2gbam as tg
import wiggle as wg
from wiggle import D, EQ, H, I, M, N, P, S, X

pytestmark = pytest.mark.gpu


def _transcript_set(tmp_path, read_type, seed):
    d = str(tmp_path / "d")
    rf.gen_dataset(d, read_type=read_type, M=40, N1=400, N0=0, seed=seed, sam=1, polyA=0)
    raw = str(tmp_path / "raw.bam")
    tg.sam_to_bam(os.path.join(d, "aln.sam"), raw, 0.0137)
    os.remove(os.path.join(d, "aln.sam"))
    wg.sort_bam(raw, os.path.join(d, "in.bam"))
    return d


SETS = {"se_q": (1, 3), "se_noq": (0, 4), "pe_q": (3, 5), "pe_noq": (2, 6)}


@pytest.mark.parametrize("key", sorted(SETS))
def test_transcript_bams(built, tmp_path, key):
    d = _transcript_set(tmp_path, *SETS[key])
    for tool, nfw in (("wig", False), ("wig", True), ("depth", False)):
        ref, ours = wg.check_same(f"{key}_{tool}{'_nfw' if nfw else ''}", d, tool, nfw)
        assert ours.returncode == 0, ours.stderr
        assert ours.output.count(b"\n") >= 40


def test_genome_bam(built, tmp_path):
    d = str(tmp_path / "d")
    rf.gen_dataset(d, read_type=3, genome=1, M=40, N1=300, N0=0, seed=5, sam=1, polyA=0)
    tg.sam_to_bam(os.path.join(d, "aln.sam"), os.path.join(d, "t.bam"), 0.0137)
    os.remove(os.path.join(d, "aln.sam"))
    tool_dir = str(tmp_path / "tool")   # the same argv[0] (it is in the @PG line) whichever executable converts
    os.makedirs(tool_dir)
    os.symlink(tg.REF_EXE if os.path.exists(tg.REF_EXE) else tg.OUR_EXE, os.path.join(tool_dir, "rsem-tbam2gbam"))
    subprocess.check_call(["./rsem-tbam2gbam", "../d/ref/r", "../d/t.bam", "../g.bam"], cwd=tool_dir,
                          stdout=subprocess.DEVNULL)
    os.remove(os.path.join(d, "t.bam"))
    wg.sort_bam(str(tmp_path / "g.bam"), os.path.join(d, "in.bam"))
    _, _, recs = bam_reader.read_bam(os.path.join(d, "in.bam"))
    spliced = {r["tags"]["XS"][1] for r in recs if "N" in r["cigar"] and "XS" in r["tags"]}
    assert spliced == {"+", "-"}   # spliced reads of genes on both strands
    for tool, nfw in (("wig", False), ("wig", True), ("depth", False)):
        ref, ours = wg.check_same(f"genome_{tool}{'_nfw' if nfw else ''}", d, tool, nfw)
        assert ours.returncode == 0, ours.stderr
        if tool == "wig":
            assert b"fixedStep" in ours.output


HAND_REFS = [("c1", 300), ("c2", 50), ("c3", 1000), ("z0", 0), ("unseen", 20), ("c4", 600), ("c5", 100)]


def _hand_records():
    rng = random.Random(11)
    r, k = [], [0]

    def add(tid, pos, cigar, aux=b"", flag=0, l_seq=None):
        k[0] += 1
        r.append(wg.record(f"r{k[0]}", flag, tid, pos, cigar, aux, l_seq))
    # c1: every CIGAR operation, ZW of every type, the first ZW only, tags before it
    add(0, 3, [(10, M), (5, EQ), (3, X), (4, D), (2, N), (6, M)], wg.zwf(0.3))
    add(0, 5, [(5, S), (10, M), (3, I), (10, M), (2, H)], b"NMi" + struct.pack("<i", 2) + b"XSA+" + wg.zwf(0.7))
    add(0, 7, [(4, M), (2, P), (4, M), (3, 9), (4, M)], b"MDZ10A5\0" + b"XBBc" + struct.pack("<I", 3) + b"\1\2\3" + wg.zwf(0.11))
    add(0, 9, [], wg.zwf(0.5), l_seq=12)                                 # CIGAR '*' on a mapped record
    add(0, 9, [(30, M)])                                                # no ZW: adds nothing
    add(0, 9, [(30, M)], b"ZWi" + struct.pack("<i", 7))                 # weight 0
    add(0, 9, [(30, M)], b"ZWZ0.9\0")                                   # weight 0
    add(0, 11, [(20, M)], wg.zwd(0.123456789012345))                    # ZW:d as raw bytes
    add(0, 12, [(20, M)], wg.zwf(0.25) + wg.zwf(100.0))                 # a second ZW after the first
    add(0, 13, [(20, M)], wg.zwf(0.5) + b"YYq\1")                       # an unknown type after the ZW is never read
    for w in (-0.3, 1e-30, 1e30, 3e-6, -1e-7, 0.004, 0.0055):
        add(0, 40 + rng.randrange(30), [(rng.randrange(5, 40), M)], wg.zwf(w))
    add(0, 270, [(30, M)], wg.zwf(0.2))                                 # ends exactly at the end of c1
    # c2: only records without ZW (readdepth prints zeros, not NA)
    add(1, 0, [(20, M)])
    add(1, 30, [(20, M)], b"XXi" + struct.pack("<i", 1))
    # c3: non-finite weights, alone and in pairs
    nan, mnan, snan = 0x7fc00000, 0xffc00000, 0x7f800123
    add(2, 10, [(5, M)], wg.zwf_bits(nan))
    add(2, 20, [(5, M)], wg.zwf_bits(mnan))
    add(2, 30, [(5, M)], wg.zwf_bits(snan))
    add(2, 40, [(5, M)], wg.zwf(float("inf")))
    add(2, 50, [(5, M)], wg.zwf(float("-inf")))
    add(2, 60, [(5, M)], wg.zwf(float("inf")))
    add(2, 60, [(5, M)], wg.zwf(float("-inf")))                         # inf + -inf: the default NaN
    add(2, 70, [(5, M)], wg.zwf(float("-inf")))
    add(2, 70, [(5, M)], wg.zwf(float("inf")))
    add(2, 80, [(5, M)], wg.zwf_bits(nan))
    add(2, 80, [(5, M)], wg.zwf_bits(mnan))                             # both NaN: the depth's sign stays
    add(2, 90, [(5, M)], wg.zwf_bits(mnan | 0x1234))
    add(2, 90, [(5, M)], wg.zwf_bits(nan | 0x55))
    add(2, 100, [(5, M)], wg.zwf(float("inf")))
    add(2, 100, [(5, M)], wg.zwf(float("inf")))
    add(2, 110, [(5, M)], wg.zwf(2.0))
    add(2, 110, [(5, M)], wg.zwf_bits(mnan))
    add(2, 110, [(5, M)], wg.zwf(1.0))
    add(2, 250, [(20, M)], wg.zwd(float("nan")))
    # z0: a target of length 0 with a record that covers nothing
    add(3, 0, [(5, S)], wg.zwf(0.5), l_seq=5)
    # c1 comes back: processed again from zero
    add(0, 100, [(40, M)], wg.zwf(0.375))
    # c4: a pileup across tile boundaries, weights whose sums depend on the order
    for _ in range(300):
        add(5, 200 + rng.randrange(120), [(rng.randrange(1, 30), M), (rng.randrange(0, 5), N), (rng.randrange(1, 30), M)],
            wg.zwf(rng.choice([0.1, 0.2, 0.3, 1e-8, 3.3, 0.0137 * rng.randrange(1, 70)])))
    # c5: ends exactly at its end
    add(6, 90, [(10, M)], wg.zwf(0.5))
    return r


def test_b_arrays_before_zw(built, tmp_path):
    """htslib 1.3's skip_aux steps over a 'B' array by aux_type2size(subtype) * count whatever the subtype: 8 for 'd',
    1 for 'A', 0 for an unknown one (only its 6-byte header), the type letter's code for 'Z' / 'H' / 'B'"""
    d = str(tmp_path / "d")
    os.makedirs(d)
    arrays = [b"XBBd" + struct.pack("<I2d", 2, 1.5, -2.5), b"XBBA" + struct.pack("<I", 3) + b"abc",
              b"XBBq" + struct.pack("<I", 5), b"XBBZ" + struct.pack("<I", 0), b"XBBf" + struct.pack("<If", 1, 0.5)]
    recs = [wg.record(f"b{i}", 0, 0, 3 * i, [(20, M)], a + wg.zwf(0.1 * (i + 1))) for i, a in enumerate(arrays)]
    recs.append(wg.record("all", 0, 0, 40, [(20, M)], b"".join(arrays) + wg.zwf(0.7)))
    wg.write_bam(os.path.join(d, "in.bam"), [("c1", 100)], recs)
    for tool in ("wig", "depth"):
        ref, ours = wg.check_same(f"b_arrays_{tool}", d, tool)
        assert ours.returncode == 0, ours.stderr
    assert ours.output.startswith(b"c1\t100\t0.1 0.1 0.1 0.3 0.3 0.3 0.6 ")


def test_failed_call_reports_no_bad_record(built):
    """a call refused for its arguments leaves stats.bad_record at -1, so that the host never takes it for a record"""
    import ctypes as C
    import rsem_b200
    from rsem_b200.capi import WigBatch, WigStats
    rec = wg.record("r", 0, 0, 0, [(5, M)], wg.zwf(0.5))
    data = np.frombuffer(rec, np.uint8).copy()
    off, run, lens = np.zeros(1, np.uint64), np.zeros(1, np.uint32), np.array([10], np.uint32)
    with rsem_b200.Context(0) as ctx:
        for continues, keep_last in ((1, 0), (0, 0)):   # continues without a resident run; then a call that succeeds
            b = WigBatch(n_records=1, n_bytes=len(data), data=data.ctypes.data_as(C.POINTER(C.c_uint8)),
                         rec_off=off.ctypes.data_as(C.POINTER(C.c_uint64)), rec_run=run.ctypes.data_as(C.POINTER(C.c_uint32)),
                         run_len=lens.ctypes.data_as(C.POINTER(C.c_uint32)), n_runs=1, continues=continues,
                         keep_last=keep_last, no_fractional_weight=0)
            out = np.zeros(10)
            got = C.c_uint64(0)
            st = WigStats(bad_record=12345)
            rc = ctx.lib.dll.rsem_b200_wig_depth(ctx._h, C.byref(b), out.ctypes.data_as(C.POINTER(C.c_double)),
                                                 C.c_uint64(10), C.byref(got), C.byref(st))
            assert st.bad_record == -1
            assert (rc != 0) == bool(continues)
        assert list(out) == [0.5] * 5 + [0.0] * 5


def _hand_set(tmp_path):
    d = str(tmp_path / "d")
    os.makedirs(d)
    wg.write_bam(os.path.join(d, "in.bam"), HAND_REFS, _hand_records())
    return d


def test_hand_written_records(built, tmp_path):
    d = _hand_set(tmp_path)
    for tool, nfw in (("wig", False), ("wig", True), ("depth", False)):
        ref, ours = wg.check_same(f"hand_{tool}{'_nfw' if nfw else ''}", d, tool, nfw)
        assert ours.returncode == 0, ours.stderr
    text = ours.output.decode()
    assert " -nan " in text and " nan " in text and " inf " in text and " -inf " in text
    lines = dict(l.split("\t", 1) for l in text.splitlines())
    assert lines["z0"] == "0\tNA" and lines["unseen"] == "20\tNA" and lines["c2"] == "50\t" + " ".join(["0"] * 50)
    assert list(lines).count("c1") == 1 and text.count("c1\t300\t") == 2   # c1 is written twice


def test_progress_lines(built, tmp_path):
    d = str(tmp_path / "d")
    os.makedirs(d)
    refs = [("a", 200000), ("b", 150000), ("c", 90000)]
    rng = np.random.default_rng(4)
    recs = []
    for tid, (_, L) in enumerate(refs):
        pos = np.sort(rng.integers(0, L - 40, 400000))
        for i, p in enumerate(pos.tolist()):
            recs.append(wg.record("q", 0, tid, p, [(36, M)], wg.zwf((i % 7) * 0.125), l_seq=36))
    wg.write_bam(os.path.join(d, "in.bam"), refs, recs)
    for tool in ("wig", "depth"):
        ref, ours = wg.check_same(f"progress_{tool}", d, tool)
        assert ours.stdout == "1000000\n"


def test_forced_batches_and_threads_give_identical_files(built, tmp_path):
    d = _hand_set(tmp_path)
    os.makedirs(tmp_path / "t")
    t = _transcript_set(tmp_path / "t", 3, 5)
    for src in (d, t):
        for tool in ("wig", "depth"):
            base = wg.run_ours(src, tool, f"base_{tool}")
            assert base.returncode == 0, base.stderr
            for i, env in enumerate(({"RSEM_B200_WIG_BATCH": "1"}, {"RSEM_B200_WIG_BATCH": "200"},
                                     {"RSEM_B200_WIG_BATCH": "3000", "RSEM_B200_IO_THREADS": "1"},
                                     {"RSEM_B200_WIG_BATCH": "777", "RSEM_B200_IO_THREADS": "8"},
                                     {"RSEM_B200_IO_THREADS": "8"})):
                p = wg.run_ours(src, tool, f"b{i}_{tool}", env=env)
                assert p.returncode == 0, p.stderr
                assert p.stdout == base.stdout and p.output == base.output, (src, tool, env)


REFUSALS = {   # key: (bad record, words of the message)
    "tid_outside_header": (wg.record("bad", 0, 2, 5, [(10, M)], wg.zwf(0.5)), "not in the header"),
    "negative_pos": (wg.record("bad", 0, 0, -3, [(10, M)], wg.zwf(0.5)), "negative position"),
    "m_past_end": (wg.record("bad", 0, 1, 45, [(2, M), (3, D), (6, M)], wg.zwf(0.5)), "past the end"),
    "unknown_aux_type": (wg.record("bad", 0, 1, 5, [(10, M)], b"XXq\1" + wg.zwf(0.5)), "unknown type"),
    "truncated_aux": (wg.record("bad", 0, 1, 5, [(10, M)], b"XXi\1\0"), "cut short"),
    "truncated_z": (wg.record("bad", 0, 1, 5, [(10, M)], b"XXZabc"), "cut short"),
}


@pytest.mark.parametrize("key", sorted(REFUSALS))
def test_refusals(built, tmp_path, key):
    bad, words = REFUSALS[key]
    refs = [("c1", 100), ("c2", 50)]
    good = [wg.record(f"g{i}", 0, i // 10, 3 * (i % 10), [(10, M)], wg.zwf(0.25)) for i in range(20)]
    d = str(tmp_path / "d")
    os.makedirs(d)
    wg.write_bam(os.path.join(d, "in.bam"), refs, good + [bad])
    c = str(tmp_path / "c")
    os.makedirs(c)
    wg.write_bam(os.path.join(c, "in.bam"), refs, good)
    for tool in ("wig", "depth"):
        clean = wg.run_ours(c, tool, tool)
        p = wg.run_ours(d, tool, tool)
        assert p.returncode == 255 and words in p.stderr and "read bad" in p.stderr, p.stderr
        assert clean.output.startswith(p.output)   # nothing past the records before the bad one
        for env in ({"RSEM_B200_WIG_BATCH": "1"},):
            q = wg.run_ours(d, tool, tool + "_b1", env=env)
            assert q.returncode == 255 and clean.output.startswith(q.output)
    if key in ("unknown_aux_type", "truncated_aux", "truncated_z"):   # not read under --no-fractional-weight
        p = wg.run_ours(d, "wig", "wig_nfw", nfw=True)
        assert p.returncode == 0, p.stderr


# ---- K11 through the C ABI ------------------------------------------------------------------------------------------
def test_kernel_sums_bit_for_bit(built):
    import rsem_b200
    rng = np.random.default_rng(7)
    lens = [700, 1000]
    n = 120000
    recs, blocks, tids = [], [], []
    for i in range(n):
        t = 0 if i < n // 2 else 1
        L = lens[t]
        a = int(rng.integers(0, L - 60))
        m1, gap, m2 = int(rng.integers(1, 30)), int(rng.integers(0, 10)), int(rng.integers(0, 20))
        w = float(rng.choice([-1.0, 1.0]) * 10.0 ** rng.uniform(-6, 6))
        cig = [(m1, M), (gap, N)] + ([(m2, M)] if m2 else [])
        recs.append(wg.record("k", 0, t, a, cig, wg.zwd(w)))
        blocks.append([(a, a + m1, w)] + ([(a + m1 + gap, a + m1 + gap + m2, w)] if m2 else []))
        tids.append(t)
    want = [np.zeros(L) for L in lens]
    for t, bl in zip(tids, blocks):
        for a, b, w in bl:
            want[t][a:b] += w
    # three calls: run A, then A continued and B, then B continued
    cuts = [0, 30000, 90000, n]
    got = []
    with rsem_b200.Context(0) as ctx:
        for c in range(3):
            rs = recs[cuts[c]:cuts[c + 1]]
            data = b"".join(rs)
            off = np.cumsum([0] + [len(r) for r in rs[:-1]]).astype(np.uint64)
            tt = tids[cuts[c]:cuts[c + 1]]
            runs = sorted(set(tt))
            rec_run = np.array([runs.index(t) for t in tt], np.uint32)
            out, st = ctx.wig_depth(data, off, rec_run, [lens[t] for t in runs], continues=c > 0, keep_last=c < 2,
                                    out_len=sum(lens))
            assert st.bad_record == -1
            got.append(out)
    a_b = np.concatenate(got)
    assert len(got[0]) == 0 and len(got[1]) == lens[0] and len(got[2]) == lens[1]
    assert np.array_equal(a_b.view(np.int64), np.concatenate(want).view(np.int64))
    # the order matters: summing the same contributions the other way round changes some bits
    rev = [np.zeros(L) for L in lens]
    for t, bl in zip(reversed(tids), reversed(blocks)):
        for a, b, w in bl:
            rev[t][a:b] += w
    assert not np.array_equal(np.concatenate(rev).view(np.int64), np.concatenate(want).view(np.int64))


def test_kernel_nan_rules(built):
    """x86 addsd with the depth as destination: NaN operands keep sign and payload (the depth's when both are NaN),
    inf + -inf is the negative default NaN, ZW:f NaNs widen quiet with their payload"""
    import rsem_b200
    cases = [  # ZW:f bit patterns added in order at one position -> the double's bits
        ([0x7fc00000], 0x7ff8000000000000),
        ([0xffc00000], 0xfff8000000000000),
        ([0x7f800123], 0x7ff8002460000000),
        ([0x7f800000, 0xff800000], 0xfff8000000000000),
        ([0xff800000, 0x7f800000], 0xfff8000000000000),
        ([0x7fc00000, 0xffc00000], 0x7ff8000000000000),
        ([0xffc01234, 0x7fc00055], 0xfff8024680000000),
        ([0x3f800000, 0xffc00000, 0x40000000], 0xfff8000000000000),
        ([0x7f800000, 0x7f800000], 0x7ff0000000000000),
    ]
    recs, rec_run = [], []
    for k, (ws, _) in enumerate(cases):
        for w in ws:
            recs.append(wg.record("n", 0, 0, k, [(1, M)], wg.zwf_bits(w)))
            rec_run.append(0)
    data = b"".join(recs)
    off = np.cumsum([0] + [len(r) for r in recs[:-1]]).astype(np.uint64)
    with rsem_b200.Context(0) as ctx:
        out, st = ctx.wig_depth(data, off, rec_run, [len(cases)])
    assert [int(x) & 0xffffffffffffffff for x in out.view(np.int64)] == [c[1] for c in cases]
