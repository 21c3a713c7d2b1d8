"""bin/rsem-run-em-batch with a small batch arena (RSEM_B200_BATCH_ARENA_BYTES) on a manifest of test_em_batch_exe_gpu: an
arena of about one sample, so the run adds, fills, drains and adds again, and an arena of 1 byte, so every sample finishes
its frozen rounds on the single-sample path.  Each sample's files match the run with the default arena at
test_em_batch_exe_gpu's tolerances (K12's counts are sums of atomic adds, so their last bits depend on the order the adds
land in), each sample runs the same rounds, and the blocks stay in manifest order; the RSEM_B200_TIMING counts show which
path each sample took, how often the arena was full and how many sample-rounds K12 ran."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import rsem_files as rf
from test_dropin_gpu import CASES
from test_em_batch_exe_gpu import EXE, _blocks, _compare, _manifest
from test_gibbs_batch_arena_exe_gpu import _fills

pytestmark = pytest.mark.gpu


def _run(root, samples, tag, rt, arena):
    d = os.path.join(root, tag)
    os.makedirs(d)
    for s, _ in samples:
        shutil.copytree(s, os.path.join(d, os.path.basename(s)))
    with open(os.path.join(d, "manifest"), "w") as f:
        for s, extra in samples:
            b = os.path.basename(s)
            f.write(" ".join([f"{b}/s", f"{b}/s.temp/s", f"{b}/s.stat/s", *extra]) + "\n")
    env = dict(os.environ, RSEM_B200_TIMING="1")
    env.pop("RSEM_B200_BATCH_ARENA_BYTES", None)
    if arena is not None:
        env["RSEM_B200_BATCH_ARENA_BYTES"] = str(arena)
    p = subprocess.run([EXE, "s0/ref/r", str(rt), "manifest", "-p", "2"], cwd=d, env=env, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    m = re.search(r"(\d+) samples in the batch, (\d+) on the single-sample path; K12 [\d.]+ ms over (\d+) sample-rounds",
                  p.stderr)
    full = re.search(r"arena full (\d+) times", p.stderr)
    assert m and full, p.stderr
    blocks = _blocks(p.stdout)
    assert [b[0].split()[2] for b in blocks] == [os.path.basename(s) + "/s" for s, _ in samples]   # manifest order
    rounds = [sum(line.startswith("ROUND = ") for line in b) for b in blocks]
    return d, rounds, (int(m.group(1)), int(m.group(2)), int(full.group(1))), int(m.group(3))


def _sample_bytes(samples, rt):
    """rsem_b200_batch_sample_bytes of each sample, None for one without alignable reads, through the library"""
    import rsem_b200
    out = []
    ctx = rsem_b200.Context(0)
    try:
        with rsem_b200.Batch(ctx, 1) as b:
            for s, _ in samples:
                path = os.path.join(s, "s.temp", "s.dat")
                if not (os.path.exists(path) and int(open(path).readline().split()[0]) > 0):
                    out.append(None)
                    continue
                row_ptr, sid = rf.read_dat(path, rt >= 2)[:2]
                out.append(b.sample_bytes(row_ptr, len(np.unique(np.abs(sid)))))
    finally:
        ctx.close()
    return out


@pytest.mark.parametrize("name", ["se_noq", "pe_q_rspd"])
def test_small_arenas_match_the_default(tmp_path, built, name):
    """the arena of the second largest sample: the largest (first) does not fit even an empty arena and finishes on the
    context, the others fill the arena in turn; K12's sample-rounds are the frozen rounds (past round 10) of the samples
    that ran in the batch"""
    rt, opts = CASES[name]
    os.makedirs(tmp_path / "in")
    samples = _manifest(tmp_path / "in", rt, opts, wide=False)
    sizes = _sample_bytes(samples, rt)
    with_reads = [b for b in sizes if b is not None]
    assert len(with_reads) == 4
    one = sorted(with_reads)[-2]
    assert sizes[0] > one and _fills(with_reads, one) >= 2    # adds, fills, drains and adds again, more than once
    base, rounds0, counts0, k12_0 = _run(str(tmp_path), samples, "default", rt, None)
    frozen = [r - 10 if b is not None else 0 for r, b in zip(rounds0, sizes)]
    assert counts0 == (4, 0, 0) and k12_0 == sum(frozen) and min(frozen[k] for k in range(4)) > 0
    fits = [b is not None and b <= one for b in sizes]
    for tag, arena, want, k12 in (("one", one, (sum(fits), 4 - sum(fits), _fills(with_reads, one)),
                                   sum(f for f, ok in zip(frozen, fits) if ok)),
                                  ("none", 1, (0, 4, 4), 0)):
        d, rounds, counts, k12_rounds = _run(str(tmp_path), samples, tag, rt, arena)
        assert counts == want and k12_rounds == k12, tag
        assert rounds == rounds0, tag
        for s, extra in samples:
            b = os.path.basename(s)
            _compare(os.path.join(d, b), os.path.join(base, b), "--gibbs-out" in extra, "-b" in extra)
