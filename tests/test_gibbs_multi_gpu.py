"""Gibbs chains split over contexts and devices give the draws and sums of one run of all chains.

Through the C ABI on one H100: a run's chains are split into contiguous ranges, each range run with
rsem_b200_gibbs_run_chains on (a) the context of the upload and (b) a second context filled by rsem_b200_gibbs_upload_from;
the count vectors and the chain-order sums (rsem_b200_gibbs_sum_chains) are bit-identical to one rsem_b200_gibbs_run.

Through bin/rsem-run-gibbs: RSEM_B200_DEVICES spreads the chains over the listed devices (each used once, never more
devices than chains); every .countvectors<t> and the result rows are byte-identical to the run on one device and to the
reference's stored output of the golden data sets.  The runs over two or more distinct devices need as many GPUs."""
import ctypes as C
import filecmp
import functools
import os
import re
import shutil
import subprocess
import tarfile

import numpy as np
import pytest

import rsem_files as rf
from rsem_b200.capi import GibbsOut, GibbsParams, RsemB200Error
from test_gibbs_gpu import Problem, _family_matrix, _run_gpu

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _matrix(N):
    """family-structured matrix: N = 1000 runs the serial kernel (N1 < 1248), N = 6000 the component-parallel one"""
    M = 150 if N < 1248 else 600
    rp, sid, val = _family_matrix(N, M, seed=N, max_family=40, junk=0.3)
    return rp, sid, val, M


def _params(pb, samples, seeds, burnin, gap, keep):
    samples = np.ascontiguousarray(samples, np.int32)
    seeds = np.ascontiguousarray(seeds, np.uint32)
    init, genes = np.ascontiguousarray(pb.init, np.int32), np.ascontiguousarray(pb.genes, np.int32)
    alpha, eel, mw = (np.ascontiguousarray(x, np.float64) for x in (pb.alpha, pb.eel, pb.mw))
    keep += [samples, seeds, init, genes, alpha, eel, mw]
    p = GibbsParams()
    p.M, p.burnin, p.gap, p.n_chains = pb.M, burnin, gap, len(samples)
    p.chain_samples = samples.ctypes.data_as(C.POINTER(C.c_int32))
    p.chain_seeds = seeds.ctypes.data_as(C.POINTER(C.c_uint32))
    p.n0, p.totc = pb.n0, pb.totc
    p.init_counts = init.ctypes.data_as(C.POINTER(C.c_int32))
    p.pseudo_counts = alpha.ctypes.data_as(C.POINTER(C.c_double))
    p.eel, p.mw = eel.ctypes.data_as(C.POINTER(C.c_double)), mw.ctypes.data_as(C.POINTER(C.c_double))
    p.n_genes = len(genes) - 1
    p.gene_start = genes.ctypes.data_as(C.POINTER(C.c_int32))
    return p


def _sums(lib, pb, p_all, acc):
    sums = [np.zeros(pb.M + 1) for _ in range(4)] + [np.zeros(len(pb.genes) - 1)]
    o = GibbsOut()
    o.sum_c, o.sum_c2, o.sum_tpm, o.sum_fpkm, o.sum_gene_c2 = (s.ctypes.data_as(C.POINTER(C.c_double)) for s in sums)
    lib.gibbs_sum_chains(p_all, acc, o)
    return sums


def _run_ranges(ctx, pb, samples, seeds, burnin, gap, ranges):
    """the chains of each range on ctx -> (count vectors, per-chain blocks, worker CTAs of each range) of all chains"""
    samples, seeds = np.asarray(samples, np.int32), np.asarray(seeds, np.uint32)
    first = np.concatenate([[0], np.cumsum(samples)])
    per = 4 * (pb.M + 1) + len(pb.genes) - 1
    cv = np.full((int(samples.sum()), pb.M + 1), -7, np.int32)
    acc = np.full((len(samples), per), np.nan)
    ctas = []
    for a, b in ranges:
        keep = []
        p = _params(pb, samples[a:b], seeds[a:b], burnin, gap, keep)
        cv_r = np.zeros((int(first[b] - first[a]), pb.M + 1), np.int32)
        acc_r = np.zeros((b - a, per))
        stats = ctx.gibbs_run_chains(p, cv_r, acc_r)
        cv[first[a]:first[b]] = cv_r
        acc[a:b] = acc_r
        ctas.append(stats.worker_ctas)
        assert stats.launches >= 1 and stats.device_ms > 0.0
    return cv, acc, ctas


SPLITS = {1: [[(0, 1)]],
          2: [[(0, 1), (1, 2)]],
          3: [[(0, 1), (1, 3)], [(0, 1), (1, 2), (2, 3)]],
          9: [[(0, 4), (4, 9)], [(0, 1), (1, 5), (5, 9)], [(0, 8), (8, 9)]]}


@pytest.mark.parametrize("alpha", ["pc0.1", "prior"])
@pytest.mark.parametrize("chains", [1, 2, 3, 9])
@pytest.mark.parametrize("N", [1000, 6000])
def test_chain_ranges_match_one_run(ctx, ctx2, N, chains, alpha, monkeypatch):
    monkeypatch.delenv("RSEM_B200_GIBBS", raising=False)
    rp, sid, val, M = _matrix(N)
    a = np.full(M + 1, 0.1) if alpha == "pc0.1" else np.random.default_rng(3).uniform(0.1, 3.0, M + 1)
    pb = Problem(rp, sid, val, M, seed=N, n0=300.0, alpha=a)
    nsamples = 2 * chains + 1 if chains > 1 else 3
    samples = [nsamples // chains + (1 if i < nsamples % chains else 0) for i in range(chains)]   # uneven by one
    seeds = np.random.default_rng(chains).integers(0, 2**32, chains, dtype=np.uint64).astype(np.uint32)
    burnin, gap = 3, 2
    cv_all, sums_all, _ = _run_gpu(ctx, rp, sid, val, M, pb.n0, pb.init, pb.alpha, pb.totc, pb.eel, pb.mw, pb.genes,
                                   burnin, gap, samples, seeds)
    assert len(set(cv_all[:, 0].tolist())) > 1   # reads move in and out of the noise transcript
    ctx2.gibbs_upload_from(ctx)
    keep = []
    p_all = _params(pb, samples, seeds, burnin, gap, keep)
    for ranges in SPLITS[chains]:
        blocks = None
        for c in (ctx, ctx2):
            cv, acc, ctas = _run_ranges(c, pb, samples, seeds, burnin, gap, ranges)
            assert all((k == 0) == (N < 1248) for k in ctas)   # serial kernel below 1248 reads, else the parallel one
            assert np.array_equal(cv, cv_all), ranges
            sums = _sums(ctx.lib, pb, p_all, acc)
            for k in range(5):
                assert np.array_equal(sums[k], sums_all[k]), (ranges, k)
            assert blocks is None or np.array_equal(acc, blocks)
            blocks = acc


def test_serial_walk_on_copied_layout(ctx, ctx2, monkeypatch):
    """RSEM_B200_GIBBS=serial on a matrix of >= 1248 reads: the serial kernel reads the copied original rows"""
    rp, sid, val, M = _matrix(6000)
    pb = Problem(rp, sid, val, M, seed=1, n0=300.0)
    samples, seeds = [2, 2, 1], [11, 12, 13]
    monkeypatch.setenv("RSEM_B200_GIBBS", "serial")
    cv_all, _, _ = _run_gpu(ctx, rp, sid, val, M, pb.n0, pb.init, pb.alpha, pb.totc, pb.eel, pb.mw, pb.genes, 2, 1, samples, seeds)
    ctx2.gibbs_upload_from(ctx)
    cv, _, ctas = _run_ranges(ctx2, pb, samples, seeds, 2, 1, [(0, 2), (2, 3)])
    assert ctas == [0, 0] and np.array_equal(cv, cv_all)


def test_upload_from_refusals(ctx, ctx2, built):
    import rsem_b200
    rp, sid, val, M = _matrix(1000)
    pb = Problem(rp, sid, val, M, seed=2, n0=300.0)
    run = lambda c: _run_gpu(c, rp, sid, val, M, pb.n0, pb.init, pb.alpha, pb.totc, pb.eel, pb.mw, pb.genes, 1, 1, [2, 1],
                             [5, 6], upload=False)[0]
    ctx.gibbs_upload(rp, sid, val, M)
    want = run(ctx)
    with rsem_b200.Context(0) as fresh, rsem_b200.Context(0) as broken:
        bad = sid.copy()
        bad[len(bad) // 2] = M + 5                                   # transcript id out of range: the upload fails
        with pytest.raises(RsemB200Error, match="out of range"):
            broken.gibbs_upload(rp, bad, val, M)
        ctx2.gibbs_upload_from(ctx)
        for src, dst, msg in ((fresh, ctx2, "no completed gibbs_upload"), (broken, ctx2, "no completed gibbs_upload"),
                              (ctx2, ctx2, "the same context"), (None, ctx2, "NULL")):
            with pytest.raises(RsemB200Error, match=msg):
                dst.gibbs_upload_from(src)
            assert np.array_equal(run(ctx2), want)               # a refused call leaves dst's matrix in place
        with pytest.raises(RsemB200Error, match="gibbs_upload must be called first"):
            run(fresh)
        fresh.gibbs_upload_from(ctx2)                             # a copy of a copy
        assert np.array_equal(run(fresh), want)
    # a later upload_from replaces the matrix dst held
    rp2, sid2, val2, M2 = _matrix(6000)
    ctx2.gibbs_upload(rp2, sid2, val2, M2)
    ctx2.gibbs_upload_from(ctx)
    assert np.array_equal(run(ctx2), want)


def test_no_reads_copied(ctx, ctx2):
    """N1 = 0: nothing but the (empty) matrix to copy; every sample is the initial counts"""
    M = 5
    init = np.array([0, 0, -1, 0, 0, 0], np.int32)
    pb = Problem(np.zeros(1, np.uint64), np.zeros(0, np.int32), np.zeros(0), M, n0=7.0, init=init)
    ctx.gibbs_upload(pb.rp, pb.sid, pb.val, M)
    ctx2.gibbs_upload_from(ctx)
    cv, _, _ = _run_ranges(ctx2, pb, [2, 1], [1, 2], 0, 2, [(0, 1), (1, 2)])
    assert (cv == init + np.array([7, 0, 0, 0, 0, 0])).all()


# ---- bin/rsem-run-gibbs -------------------------------------------------------------------------------------------------------
GOLDEN = dict(burnin=10, nsamples=6, gap=2, threads=2, seed=4242)   # the reference run stored with each golden data set


def _golden(tmp_path, name):
    """a golden data set as rsem-calculate-expression leaves it before rsem-run-gibbs (the reference's 20-round EM outputs)"""
    d = tmp_path / name
    with tarfile.open(os.path.join(rf.ROOT, "tests", "golden", name + ".tar.gz")) as t:
        t.extractall(tmp_path / "x", filter="data")
    src = tmp_path / "x" / name
    shutil.copytree(src / "ref", d / "ref")
    os.makedirs(d / "s.temp")
    os.makedirs(d / "s.stat")
    shutil.copy(src / "s.temp" / "s.omit", d / "s.temp" / "s.omit")
    for f, to in (("ofg20", "s.temp/s.ofg"), ("model20", "s.stat/s.model"), ("iso_res20", "s.temp/s.iso_res"),
                  ("gene_res20", "s.temp/s.gene_res")):
        shutil.copy(src / "out" / f, d / to)
    shutil.copytree(src / "out", tmp_path / (name + ".stored"))
    shutil.rmtree(tmp_path / "x")
    M = int(open(d / "ref" / "r.ti").readline().split()[0])
    open(d / "prior.txt", "w").write("".join(f"{0.1 + (i % 7) * 0.4:.2f} a comment\n" for i in range(M)))
    return str(d)


def _gibbs(base, key, devices, burnin, nsamples, gap, threads, seed, extra=(), which="ours"):
    d = rf.clone(base, base + "." + key)
    env = {k: v for k, v in os.environ.items() if not k.startswith("RSEM_B200_DEVICE")}
    env["RSEM_B200_TIMING"] = "1"
    if devices is not None:
        env["RSEM_B200_DEVICES"] = devices
    exe = os.path.join(rf.REF_DIR if which == "ref" else rf.BIN_DIR, "rsem-run-gibbs")
    cmd = [exe, "ref/r", "s.temp/s", "s.stat/s", str(burnin), str(nsamples), str(gap), "-p", str(threads), "--seed", str(seed),
           *extra]
    p = subprocess.run(cmd, cwd=d, env=env, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-2000:]
    used = [int(x) for x in re.findall(r"rsem-run-gibbs timing: device (\d+):", p.stderr)]
    return d, p, used


def _same_files(a, b, threads):
    for t in range(threads):
        assert filecmp.cmp(f"{a}/s.temp/s.countvectors{t}", f"{b}/s.temp/s.countvectors{t}", shallow=False), t
    assert not os.path.exists(f"{a}/s.temp/s.countvectors{threads}")
    for f in ("s.iso_res", "s.gene_res"):
        assert filecmp.cmp(f"{a}/s.temp/{f}", f"{b}/s.temp/{f}", shallow=False), f


def _n_gpus():
    import rsem_b200
    return rsem_b200.load_library().device_count()


@pytest.mark.parametrize("name", ["pe_q_rspd", "se_noq"])
def test_tool_golden_one_device(tmp_path, built, name):
    """the stored reference run of a golden data set, on one device however it is named: '0,0' uses card 0 once (no two
    cooperative grids on one card); stdout is the same whatever the list"""
    base = _golden(tmp_path, name)
    stored = tmp_path / (name + ".stored")
    outs = []
    for devices in (None, "0", "0,0"):
        d, p, used = _gibbs(base, str(devices).replace(",", "_"), devices, **GOLDEN)
        assert used == [0]
        outs.append(p.stdout)
        for t in range(GOLDEN["threads"]):
            assert filecmp.cmp(f"{d}/s.temp/s.countvectors{t}", stored / f"countvectors{t}", shallow=False)
        assert filecmp.cmp(f"{d}/s.temp/s.iso_res", stored / "iso_res_gibbs", shallow=False)
        assert filecmp.cmp(f"{d}/s.temp/s.gene_res", stored / "gene_res_gibbs", shallow=False)
    assert outs[0] == outs[1] == outs[2] and "Gibbs finished!" in outs[0]


def test_tool_one_chain_two_devices(tmp_path, built):
    """-p 1 with two devices listed: one chain, one device (the second is never opened)"""
    base = _golden(tmp_path, "se_noq")
    one, _, used1 = _gibbs(base, "one", None, 10, 5, 2, 1, 77)
    two, _, used2 = _gibbs(base, "two", "0,1", 10, 5, 2, 1, 77)
    assert used1 == [0] and used2 == [0]
    _same_files(one, two, 1)


CASES = [  # (data set, burnin, nsamples, gap, -p, seed, extra arguments)
    ("pe_q_rspd", 10, 6, 2, 2, 4242, []),
    ("se_noq", 20, 9, 1, 3, 5, []),
    ("pe_q_rspd", 5, 19, 3, 8, 1, []),
    ("se_noq", 10, 6, 1, 2, 99, ["--pseudo-count", "0.1"]),
    ("se_q_polyA", 10, 7, 2, 3, 99, ["--prior", "prior.txt"]),
    ("pe_noq", 0, 30, 1, 8, 12345, []),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_tool_devices_match_one_device(tmp_path, built, case):
    n = _n_gpus()
    if n < 2:
        pytest.skip("needs two GPUs")
    name, burnin, nsamples, gap, threads, seed, extra = CASES[case]
    base = _golden(tmp_path, name)
    one, _, used = _gibbs(base, "one", None, burnin, nsamples, gap, threads, seed, extra)
    assert used == [0]
    lists = ["0,1"] + ([",".join(str(i) for i in range(n))] if n > 2 else []) + ["1,0,1"]
    for devs in lists:
        d, p, used = _gibbs(base, devs.replace(",", "_"), devs, burnin, nsamples, gap, threads, seed, extra)
        want = list(dict.fromkeys(int(x) for x in devs.split(",")))[:threads]
        assert used == want, (devs, used)
        _same_files(d, one, threads)
    if rf.have_ref():
        ref, _, _ = _gibbs(base, "ref", None, burnin, nsamples, gap, threads, seed, extra, which="ref")
        _same_files(d, ref, threads)


def test_tool_devices_then_credibility_intervals(tmp_path, built):
    """rsem-calculate-credibility-intervals on the count vectors of a two-device run: its rows are the reference's"""
    if _n_gpus() < 2:
        pytest.skip("needs two GPUs")
    import test_ci_gpu
    os.environ["RSEM_B200_DEVICES"] = "0,1"
    try:
        d = test_ci_gpu._dataset(tmp_path, "ci_p3_30", "pe_q_rspd", 30, 3)
    finally:
        del os.environ["RSEM_B200_DEVICES"]
    test_ci_gpu._compare(tmp_path, d, "ci_p3_30", 0.95, 30, 20, 3, 5)


@pytest.fixture(scope="module")
def ctx(built):
    import rsem_b200
    c = rsem_b200.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ctx2(built):
    """a second context on the same device, filled by gibbs_upload_from"""
    import rsem_b200
    c = rsem_b200.Context(0)
    yield c
    c.close()
