"""bin/rsem-calculate-credibility-intervals-batch against bin/rsem-calculate-credibility-intervals: every manifest line
must append the rows a single run of that line appends to imd.iso_res / imd.gene_res (and imd.allele_res), byte for
byte, and print the same stdout block (a multiset of lines where -p > 1: the sampler threads print side by side).
Lines that repeat a stored case of test_ci_gpu.py must also give that case's reference digests.  Then the lanes, K8's
kept buffers across resident and host-memory samples, quiet lines and lines without --seed, a count-vector file that
does not hold its line's vectors, and the kept buffers through rsem_b200.Context."""
import ctypes
import hashlib
import os
import shutil
import subprocess

import numpy as np
import pytest

import ci_phase2 as cp
import rsem_files as rf
import test_ci_gpu as single
from rsem_b200.capi import CiParams, _p

pytestmark = pytest.mark.gpu

BATCH = os.path.join(rf.BIN_DIR, "rsem-calculate-credibility-intervals-batch")
RESULTS = ("s.iso_res", "s.gene_res", "s.allele_res")


def _vectors(d):
    """the count vectors of the rsem-run-gibbs run in d, one text line each"""
    out = []
    for t in range(8):
        f = d / "s.temp" / f"s.countvectors{t}"
        if os.path.exists(f):
            out += [x for x in open(f).read().split("\n") if x.strip()]
    return out


def _cohort(tmp_path, d, lines):
    """a directory with d's reference and model and one sample directory per line.  A line is (confidence, nCV, nSpC,
    -p, further options), its count vectors the first nCV of d's split over min(-p, nCV) files; or ("copy", the
    arguments after statName) for a copy of d's own s.temp, as a stored case of test_ci_gpu.py runs it.
    -> (root, manifest text)"""
    root = tmp_path / "cohort"
    shutil.copytree(d / "ref", root / "ref")
    shutil.copytree(d / "s.stat", root / "st")
    vecs = _vectors(d)
    text = []
    for j, line in enumerate(lines, 1):
        sd = root / f"l{j}"
        if line[0] == "copy":
            shutil.copytree(d / "s.temp", sd)
            text.append(f"l{j}/s st/s {line[1]}")
            continue
        conf, ncv, nspc, threads, extra = line
        os.makedirs(sd)
        k = min(threads, ncv)
        for t in range(k):   # the first ncv vectors, split as evenly as they go
            part = vecs[t * ncv // k:(t + 1) * ncv // k]
            open(sd / f"s.countvectors{t}", "w").write("".join(x + "\n" for x in part))
        text.append(f"l{j}/s st/s {conf} {ncv} {nspc} 1024 -p {threads} {extra}")
    return root, "".join(x + "\n" for x in text)


def _blocks(stdout):
    """batch stdout -> {line number: block}"""
    out, cur = {}, None
    for ln in stdout.splitlines(keepends=True):
        if ln.startswith("== sample "):
            cur = int(ln.rsplit("line ", 1)[1].rstrip(")\n"))
            out[cur] = ""
        else:
            out[cur] += ln
    return out


def _files(root, n):
    return {(j, f): open(root / f"l{j}" / f, "rb").read() for j in range(1, n + 1) for f in RESULTS
            if os.path.exists(root / f"l{j}" / f)}


def _run_batch(root, manifest, env=None, extra=()):
    open(root / "manifest", "w").write(manifest)
    return subprocess.run([BATCH, "ref/r", "manifest", *extra], cwd=root, capture_output=True, text=True,
                          env={**os.environ, **(env or {})})


def _against_single(tmp_path, root, manifest, env=None):
    """runs the batch in a copy of root and the single tool line by line in another; asserts the same files and
    blocks -> (batch process, batch copy)"""
    b, s = tmp_path / "batch", tmp_path / "single"
    shutil.copytree(root, b)
    shutil.copytree(root, s)
    p = _run_batch(b, manifest, env)
    assert p.returncode == 0, p.stderr
    blocks = _blocks(p.stdout)
    lines = [x for x in manifest.split("\n") if x.strip()]
    for j, line in enumerate(lines, 1):
        q = subprocess.run([single.BIN, "ref/r", *line.split()], cwd=s, capture_output=True, text=True,
                           env={**os.environ, **(env or {})})
        assert q.returncode == 0, q.stderr
        if " -p 1 " in line + " ":
            assert blocks[j] == q.stdout, line
        else:
            assert sorted(blocks[j].splitlines()) == sorted(q.stdout.splitlines()), line
    assert _files(b, len(lines)) == _files(s, len(lines))
    return p, b


def _stored_digests(tmp_path, d, key, args):
    ref = tmp_path / (key + ".ref")
    shutil.copytree(d, ref)
    r = rf.reference_run(key, str(ref), lambda: subprocess.run([single.REF_BIN, "ref/r", "s.temp/s", "s.stat/s", *args],
                                                               cwd=ref, capture_output=True, text=True), digests_only=True)
    assert r.returncode == 0, r.stderr
    return {os.path.basename(k): v for k, v in r.digests.items() if os.path.basename(k) in RESULTS}


def _digests(sd):
    return {f: hashlib.sha256(open(sd / f, "rb").read()).hexdigest() for f in RESULTS if os.path.exists(sd / f)}


# -p 1, 2, 3 and above nCV; pseudo-counts 1, 0.1, 0.001; nSamples % 4 = 0, 3, 1, 2; confidence 0.95 and 0.5
VARIED = [(0.95, 40, 4, 1, "--pseudo-count 1 --seed 3"),
          (0.5, 39, 1, 2, "--pseudo-count 0.1 --seed 4"),
          (0.95, 37, 1, 3, "--pseudo-count 0.001 --seed 5"),
          (0.5, 2, 19, 5, "--seed 6")]


@pytest.mark.parametrize("name", ["se_noq", "se_q_polyA", "pe_noq", "pe_q_rspd"])
def test_lines_match_single_runs(tmp_path, name):
    d = single._dataset(tmp_path, f"ci_{name}", name, 40, 2)
    stored = "0.95 40 25 1024 -p 2 --seed 11"   # test_ci_gpu.py's test_model_types
    root, manifest = _cohort(tmp_path, d, [("copy", stored)] + VARIED)
    p, b = _against_single(tmp_path, root, manifest)
    assert _digests(b / "l1") == _stored_digests(tmp_path, d, f"ci_{name}", stored.split())


def test_allele_specific_reference(tmp_path):
    d = single._dataset(tmp_path, "ci_allele", "se_q_rspd", 20, 1, alleles=True)
    stored = "0.95 20 30 1024 -p 1 --seed 9"   # test_ci_gpu.py's test_allele_specific_reference
    root, manifest = _cohort(tmp_path, d, [("copy", stored), (0.95, 20, 10, 2, "--seed 2"), (0.5, 19, 3, 1, "--seed 5")])
    p, b = _against_single(tmp_path, root, manifest)
    assert os.path.exists(b / "l2" / "s.allele_res")
    assert _digests(b / "l1") == _stored_digests(tmp_path, d, "ci_allele", stored.split())


def test_lanes(tmp_path):
    d = single._dataset(tmp_path, "ci_lanes", "pe_q_rspd", 40, 2)
    root, manifest = _cohort(tmp_path, d, VARIED + [(0.95, 40, 10, 2, "--seed 8"), (0.95, 30, 3, 1, "--seed 9")])
    n = 6
    p, one = _against_single(tmp_path, root, manifest)
    want = _files(one, n)
    sets = ["0,0", "0,0,0"]
    import torch
    if torch.cuda.device_count() >= 2:
        sets.append("0,1")
    for devices in sets:
        run = tmp_path / ("lanes" + devices.replace(",", ""))
        shutil.copytree(root, run)
        q = _run_batch(run, manifest, {"RSEM_B200_DEVICES": devices})
        assert q.returncode == 0, q.stderr
        assert _files(run, n) == want, devices
        assert {j: sorted(x.splitlines()) for j, x in _blocks(q.stdout).items()} == \
            {j: sorted(x.splitlines()) for j, x in _blocks(p.stdout).items()}


def test_kept_buffers_across_paths(tmp_path):
    """one lane, one budget: the sample matrix on the device, in host memory, on the device, then a larger one on the
    device; every file as the single tool writes it with the same budget"""
    d = single._dataset(tmp_path, "ci_kept", "pe_q_rspd", 40, 2)
    M = int(open(d / "ref" / "r.ti").readline().split()[0])
    mr = single._max_gene_rows(d)
    resident = lambda n: n * M * 4 + n * 20 + (1 << 20) + mr * n * 8
    host_ok = lambda n: n * 20 + (1 << 20) + mr * n * 12
    budget = resident(400)
    assert resident(560) > budget >= host_ok(560)
    lines = [(0.95, 40, 5, 2, "--seed 1"), (0.95, 40, 14, 2, "--seed 2"), (0.5, 40, 5, 1, "--seed 3"),
             (0.95, 40, 10, 3, "--seed 4")]
    root, manifest = _cohort(tmp_path, d, lines)
    p, _ = _against_single(tmp_path, root, manifest, {"RSEM_B200_CI_DEVICE_BYTES": str(budget), "RSEM_B200_TIMING": "1"})
    assert "4 samples (1 with the matrix in host memory)" in p.stderr, p.stderr


def test_quiet_and_unseeded_lines(tmp_path):
    d = single._dataset(tmp_path, "ci_quiet", "pe_noq", 40, 2)
    root, manifest = _cohort(tmp_path, d, [(0.95, 40, 10, 1, "--seed 1"), (0.95, 40, 10, 2, "-q --seed 2"),
                                           (0.95, 40, 10, 1, "")])
    p = _run_batch(rf.clone(root, tmp_path / "a"), manifest)
    assert p.returncode == 0, p.stderr
    blocks = _blocks(p.stdout)
    assert blocks[2] == ""
    s = rf.clone(root, tmp_path / "s")
    q = subprocess.run([single.BIN, "ref/r", "l3/s", "st/s", "0.95", "40", "10", "1024", "-p", "1", "--seed", "7"], cwd=s,
                       capture_output=True, text=True)
    assert q.returncode == 0, q.stderr
    assert blocks[3] == q.stdout   # the progress lines do not depend on the seed
    for f in ("s.iso_res", "s.gene_res"):   # six rows, as many columns as the seeded run's
        got, want = open(tmp_path / "a" / "l3" / f).read().split("\n"), open(s / "l3" / f).read().split("\n")
        assert len(got) == len(want) == 7 and [len(x.split("\t")) for x in got] == [len(x.split("\t")) for x in want]
    # -q drops every block; the seeded lines' rows do not change
    b = rf.clone(root, tmp_path / "b")
    r = _run_batch(b, manifest, extra=("-q",))
    assert r.returncode == 0 and r.stdout == "", r.stderr
    a = _files(tmp_path / "a", 2)
    assert {k: v for k, v in _files(b, 2).items()} == a


def test_count_vectors_short_of_the_line(tmp_path):
    """the files of line 2 hold 40 vectors, the line says 41: known only once they are parsed, so a lane reports it"""
    d = single._dataset(tmp_path, "ci_short", "pe_noq", 40, 2)
    root, manifest = _cohort(tmp_path, d, [(0.95, 40, 5, 1, "--seed 1"), (0.95, 40, 5, 1, "--seed 2")])
    manifest = manifest.replace("l2/s st/s 0.95 40", "l2/s st/s 0.95 41")
    p = _run_batch(root, manifest)
    assert p.returncode == 255
    assert ("rsem-calculate-credibility-intervals-batch: device 0, sample l2/s (manifest line 2): The count-vector files "
            "hold 40 count vectors, not nCV = 41!") in p.stderr, p.stderr
    assert not os.path.exists(root / "l2" / "s.iso_res")


# ---- K8's kept buffers through rsem_b200.Context ---------------------------------------------------------------------
C_INT = ctypes.c_int32


def _case(seed, M_genes, n):
    rng = np.random.default_rng(seed)
    sizes = rng.integers(1, 5, M_genes)
    gene_start = np.concatenate([[1], 1 + np.cumsum(sizes)]).astype(np.int32)
    M = int(gene_start[-1] - 1)
    tm = (rng.standard_exponential((M, n), dtype=np.float32) ** 3 * np.float32(40)).astype(np.float32)
    l_bars = np.exp(rng.uniform(np.log(30.0), np.log(1e4), n)).astype(np.float32)
    iso = None
    if seed % 2:   # allele-specific: pairs of transcripts inside a gene form an isoform
        iso = [1]
        for g in range(len(gene_start) - 1):
            a, b = int(gene_start[g]), int(gene_start[g + 1])
            for j in range(a, b, 2):
                iso.append(min(j + 2, b))
        iso = np.array(iso, np.int32)
    return gene_start, tm, l_bars, iso


def _ci(ctx, gene_start, tm, l_bars, threshold, budget, iso):
    M, n = tm.shape
    pg = np.array([0, len(gene_start) - 1], np.int32)
    p = CiParams(M=M, n_genes=len(gene_start) - 1, gene_start=_p(gene_start, C_INT),
                 n_isoforms=0 if iso is None else len(iso) - 1, n_parts=1, isoform_start=_p(iso, C_INT),
                 part_gene_start=_p(pg, C_INT), n_samples=n, threshold=threshold, device_budget=budget)
    ctx.ci_begin(p)
    for a in range(0, n, 700):
        ctx.ci_push(np.ascontiguousarray(tm[:, a:a + 700].T), l_bars[a:a + 700], a)
    tr, ge, io, st = ctx.ci_end(M, len(gene_start) - 1, 0 if iso is None else len(iso) - 1)
    return tr.view(np.uint32).copy(), ge.view(np.uint32).copy(), io.view(np.uint32).copy(), st


def _runs():
    """(case, budget): growing and shrinking M and n, the default budget, budgets that force host memory and blocks"""
    out = []
    for k, (genes, n) in enumerate([(300, 2000), (40, 500), (900, 3000), (300, 2000), (50, 6000), (900, 3000)]):
        gene_start, tm, l_bars, iso = _case(k, genes, n)
        M = tm.shape[0]
        mr = int(cp.gene_rows(gene_start.tolist()).max())
        budgets = [0, n * M * 4 + n * 20 + (1 << 20) + 3 * mr * n * 8, n * 20 + (1 << 20) + 2 * mr * n * 12 + n * 4]
        out.append(((gene_start, tm, l_bars, iso), budgets[k % 3]))
    return out


def test_context_runs_match_fresh_contexts(built):
    import rsem_b200
    runs = _runs()
    with rsem_b200.Context(0) as ctx:
        kept = [_ci(ctx, *c[:3], cp.threshold(0.95, c[1].shape[1]), b, c[3]) for c, b in runs]
    paths = set()
    for (c, b), got in zip(runs, kept):
        with rsem_b200.Context(0) as fresh:
            want = _ci(fresh, *c[:3], cp.threshold(0.95, c[1].shape[1]), b, c[3])
        for g, w in zip(got[:3], want[:3]):
            assert np.array_equal(g, w)
        assert (got[3].resident, got[3].blocks) == (want[3].resident, want[3].blocks)
        paths.add((got[3].resident, got[3].blocks > 1))
    assert {(1, False), (0, True)} <= paths, paths


def test_context_same_shape_keeps_memory(built):
    import torch
    import rsem_b200
    (c, b), = [r for r in _runs()[:1]]
    thr = cp.threshold(0.95, c[1].shape[1])
    with rsem_b200.Context(0) as ctx:
        _ci(ctx, *c[:3], thr, b, c[3])
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(0)[0]
        M, n = c[1].shape
        pg = np.array([0, len(c[0]) - 1], np.int32)
        p = CiParams(M=M, n_genes=len(c[0]) - 1, gene_start=_p(c[0], C_INT), n_isoforms=0, n_parts=1,
                     isoform_start=_p(None, C_INT), part_gene_start=_p(pg, C_INT), n_samples=n, threshold=thr,
                     device_budget=b)
        ctx.ci_begin(p)
        ctx.ci_push(np.ascontiguousarray(c[1].T), c[2], 0)
        free1 = torch.cuda.mem_get_info(0)[0]
        ctx.ci_end(M, len(c[0]) - 1)
        free2 = torch.cuda.mem_get_info(0)[0]
    assert free0 == free1 == free2, (free0, free1, free2)
