"""bin/rsem-run-em-batch against bin/rsem-run-em run once per sample (itself held to the reference by test_dropin_gpu),
at test_dropin_gpu's tolerances, and against the reference binary where oracle/_ref is built.

Manifests of 4-6 samples share one reference (gen_dataset --sample-seed) and mix sizes, read types, -b (with and
without --sampling), --gibbs-out, --append-names, a sample without alignable reads and one whose compact transcript set
is too large for the batch layout (it finishes on the single-sample path)."""
import filecmp
import os
import subprocess

import numpy as np
import pytest

import rsem_files as rf
from test_dropin_gpu import CASES, _num_rows_close

pytestmark = pytest.mark.gpu

EXE = os.path.join(rf.BIN_DIR, "rsem-run-em-batch")


def _manifest(root, rt, opts, wide):
    """[(dir, manifest options)] of one manifest; the first sample is the largest, so it finishes last"""
    base = dict(opts, seed=7)
    if wide:   # every sample shares the reference of the wide one
        base.update(M=26000, avg_family=1)
    specs = [
        (dict(base, N1=opts["N1"] * 4), []),
        (dict(base, N1=max(opts["N1"] // 4, 50), sam=1), ["-b", "{d}/aln.sam", "0", "--gibbs-out"]),
        (dict(base, sam=1, expressed_frac=0.3), ["-b", "{d}/aln.sam", "0", "--sampling", "--seed", "4242"]),
        (dict(base, N1=opts["N1"] // 2), ["--append-names", "--gibbs-out"]),
        (dict(base, N1=0, N0=40, sam=1), ["-b", "{d}/aln.sam", "0"]),
    ]
    if wide:   # more than 12287 distinct transcripts: outside the batch layout
        specs.append((dict(base, N1=120000, N0=100), ["--gibbs-out"]))
    out = []
    for k, (gen, extra) in enumerate(specs):
        d = str(root / f"s{k}")
        rf.gen_dataset(d, read_type=rt, sample_seed=100 + k, **gen)
        out.append((d, [x.format(d=os.path.basename(d)) for x in extra]))
    if wide:
        _, sid = rf.read_dat(os.path.join(out[-1][0], "s.temp", "s.dat"), rt >= 2)[:2]
        assert len(np.unique(np.abs(sid))) > 12287
    return out


def _single(d, name, rt, extra, rounds):
    """bin/rsem-run-em on one sample, in a copy d of its directory `name`"""
    env = dict(os.environ)
    if rounds is not None:
        env["RSEM_MAX_ROUND"], env["RSEM_MIN_ROUND"] = str(rounds), str(min(20, rounds))
    cmd = [os.path.join(rf.BIN_DIR, "rsem-run-em"), "ref/r", str(rt), "s", "s.temp/s", "s.stat/s", "-p", "2"]
    cmd += [x.replace(name + "/", "") for x in extra]
    return subprocess.run(cmd, cwd=d, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, check=True)


def _compare(a, b, has_ofg, has_bam):
    ta, tb = os.path.join(a, "s.stat", "s.theta"), os.path.join(b, "s.stat", "s.theta")
    if os.path.getsize(tb) == 0:
        assert os.path.getsize(ta) == 0
    else:
        for x, y in zip(rf.read_theta(ta), rf.read_theta(tb)):
            assert rf.close_rel(x, y, 1e-6), rf.max_rel(x, y)
        mr, mo = rf.read_tokens(os.path.join(b, "s.stat", "s.model")), rf.read_tokens(os.path.join(a, "s.stat", "s.model"))
        assert mr.shape == mo.shape and np.all(np.abs(mo - mr) <= 1e-9 + 1e-6 * np.abs(mr))
    for f in ("iso_res", "gene_res"):
        _num_rows_close(rf.read_res(os.path.join(a, "s.temp", "s." + f)), rf.read_res(os.path.join(b, "s.temp", "s." + f)))
    if has_ofg:
        Mr, N0r, rp_r, sid_r, c_r = rf.read_ofg(os.path.join(b, "s.temp", "s.ofg"))
        Mo, N0o, rp_o, sid_o, c_o = rf.read_ofg(os.path.join(a, "s.temp", "s.ofg"))
        assert (Mr, N0r) == (Mo, N0o) and np.array_equal(rp_r, rp_o) and np.array_equal(sid_r, sid_o)
        assert np.all(np.abs(c_o - c_r) <= 1e-6 * np.abs(c_r))
    if has_bam and os.path.getsize(tb) == 0:   # no alignable reads: the input is copied as it is (EM.cpp:627-633)
        assert filecmp.cmp(os.path.join(a, "s.transcript.bam"), os.path.join(b, "s.transcript.bam"), shallow=False)
    elif has_bam:
        from bam_reader import read_bam
        ta_, ra_, xa = read_bam(os.path.join(a, "s.transcript.bam"))
        tb_, rb_, xb = read_bam(os.path.join(b, "s.transcript.bam"))
        assert (ta_, ra_) == (tb_, rb_) and len(xa) == len(xb)
        for x, y in zip(xa, xb):
            zx, zy = x["tags"].pop("ZW", None), y["tags"].pop("ZW", None)
            assert (zx is None) == (zy is None)
            if zy is not None:
                assert abs(zx[1] - zy[1]) <= 1e-6 + 1e-6 * abs(zy[1])
                assert abs(x["mapq"] - y["mapq"]) <= (0 if zx[1] == zy[1] else 1)
                x["mapq"] = y["mapq"]
            assert x == y


def _blocks(stdout):
    blocks, cur = [], None
    for line in stdout.splitlines():
        if line.startswith("== sample "):
            cur = [line]
            blocks.append(cur)
        elif cur is not None:
            cur.append(line)
    return blocks


@pytest.mark.parametrize("rounds", [13, 3, None])
@pytest.mark.parametrize("name", ["se_noq", "se_q_rspd_polyA", "pe_noq", "pe_q_rspd"])
def test_batch_matches_single_sample_runs(tmp_path, built, name, rounds):
    rt, opts = CASES[name]
    samples = _manifest(tmp_path, rt, opts, wide=(name == "se_noq" and rounds is None))
    singles = []
    for d, extra in samples:
        s = rf.clone(d, d + "_single")
        singles.append((s, _single(s, os.path.basename(d), rt, extra, rounds)))
    with open(tmp_path / "manifest", "w") as f:
        for d, extra in samples:
            b = os.path.basename(d)
            f.write(" ".join([f"{b}/s", f"{b}/s.temp/s", f"{b}/s.stat/s", *extra]) + "\n\n")
    env = dict(os.environ)
    if rounds is not None:
        env["RSEM_MAX_ROUND"], env["RSEM_MIN_ROUND"] = str(rounds), str(min(20, rounds))
    p = subprocess.run([EXE, "s0/ref/r", str(rt), "manifest", "-p", "2"], cwd=tmp_path, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    assert p.stdout.rstrip().splitlines()[-1].startswith("Time Used for EM.cpp")
    blocks = _blocks(p.stdout)
    assert [b[0].split()[2] for b in blocks] == [os.path.basename(d) + "/s" for d, _ in samples]   # manifest order
    for (d, extra), (s, ps), blk in zip(samples, singles, blocks):
        rounds_b = [l for l in blk if l.startswith("ROUND = ")]
        rounds_s = [l for l in ps.stdout.splitlines() if l.startswith("ROUND = ")]
        assert len(rounds_b) == len(rounds_s)
        if rounds is not None and rounds_s:
            assert len(rounds_s) == rounds
        _compare(d, s, "--gibbs-out" in extra, "-b" in extra)
    if rf.have_ref() and rounds is not None:   # the largest sample against the reference binary itself
        ref = rf.clone(samples[0][0], samples[0][0] + "_ref")
        rf.run_em(ref, rt, "ref", rounds=rounds, threads=2, gibbs_out=False)
        _compare(samples[0][0], ref, False, False)
