"""bin/rsem-run-gibbs-batch with a small batch arena (RSEM_B200_BATCH_ARENA_BYTES) on test_gibbs_batch_exe_gpu's samples:
an arena of about one sample, so the run adds, fills, drains and adds again, and an arena of 1 byte, so every sample takes
the single-sample path.  Every file and standard output are byte-identical to the run with the default arena; the
RSEM_B200_TIMING counts show which path each sample took and how often the arena was full."""
import filecmp
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import rsem_files as rf
from rsem_b200.capi import GIBBS_BATCH_MAX_READS, GIBBS_BATCH_MIN_READS
from test_gibbs_batch_exe_gpu import EXE, M, SPECS, _files, _threads, samples  # noqa: F401  (samples: the module's fixture)

pytestmark = pytest.mark.gpu


def _run(root, tag, arena):
    d = os.path.join(root, tag)
    shutil.copytree(root + "/in", d)
    with open(os.path.join(d, "manifest"), "w") as f:
        f.write("".join(f"d{k}/s.temp/s d{k}/s.stat/s {args}\n" for k, (_, args) in enumerate(SPECS)))
    env = dict(os.environ, RSEM_B200_TIMING="1")
    env.pop("RSEM_B200_BATCH_ARENA_BYTES", None)
    if arena is not None:
        env["RSEM_B200_BATCH_ARENA_BYTES"] = str(arena)
    p = subprocess.run([EXE, "d0/ref/r", "manifest"], cwd=d, env=env, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    m = re.search(r"(\d+) samples in the batch, (\d+) on the single-sample path", p.stderr)
    full = re.search(r"arena full (\d+) times", p.stderr)
    assert m and full, p.stderr
    return d, p.stdout, (int(m.group(1)), int(m.group(2)), int(full.group(1)))


def _sample_bytes(root):
    """gibbs_batch_sample_bytes of each manifest line (None outside the size rule), through the library"""
    import rsem_b200
    from rsem_b200.capi import GibbsBatch
    n_genes = len(np.loadtxt(os.path.join(root, "d0", "ref", "r.grp"), dtype=np.int64, ndmin=1)) - 1
    out = []
    ctx = rsem_b200.Context(0)
    try:
        with GibbsBatch(ctx, 1) as b:
            for k, (_, args) in enumerate(SPECS):
                _, _, rp, sid, _ = rf.read_ofg(os.path.join(root, f"d{k}", "s.temp", "s.ofg"))
                N1 = len(rp) - 1
                a = args.split()
                ok = GIBBS_BATCH_MIN_READS <= N1 <= GIBBS_BATCH_MAX_READS
                out.append(b.sample_bytes(N1, len(sid), M, n_genes, int(a[1]), _threads(args)) if ok else None)
    finally:
        ctx.close()
    return out


def _fills(sizes, capacity):
    """times the executable finds the arena full: before an add that does not fit, it runs and empties the batch"""
    used = full = 0
    for b in sizes:
        if used + b > capacity:
            full += 1
            used = 0
        if b <= capacity:
            used += b
    return full


def test_small_arenas_match_the_default(samples, tmp_path):
    root = str(tmp_path)
    shutil.copytree(samples, root + "/in")
    sizes = _sample_bytes(root + "/in")
    batched = [b for b in sizes if b is not None]
    assert len(batched) == 4
    one = max(batched)                                       # the largest sample alone fills it
    assert _fills(batched, one) >= 2                        # adds, fills, drains and adds again, more than once
    base, out0, counts0 = _run(root, "default", None)
    assert counts0 == (4, 2, 0)
    for tag, arena, want in (("one", one, (4, 2, _fills(batched, one))), ("none", 1, (0, 6, 4))):
        d, out, counts = _run(root, tag, arena)
        assert counts == want, tag
        assert out == out0, tag                                # the same blocks, in manifest order
        for k, (_, args) in enumerate(SPECS):
            for f in _files(f"d{k}", _threads(args)):
                assert filecmp.cmp(os.path.join(d, f"d{k}", f), os.path.join(base, f"d{k}", f), shallow=False), (tag, k, f)
