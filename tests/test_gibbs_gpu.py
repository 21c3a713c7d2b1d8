"""K5/K6 through the C ABI against the CPU oracle: same seeds -> the same draws (count vectors bit-identical),
including matrices where reads move in and out of the noise transcript all the time (the case the
component-parallel sampler has to roll back and redo).

Every case runs under each walk it applies to (WALKS) and asserts that it reached the edge it is about: component
sizes from the read x transcript graph (scipy), row lengths and repeated ids from the CSR, launch waves from the
context's launch counter, worker CTAs and passes from the RSEM_B200_TIMING lines of the parallel path."""
import ctypes as C
import re

import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

import synth
from rsem_b200.capi import GibbsOut, GibbsParams, RsemB200Error

pytestmark = pytest.mark.gpu

EPS = 1e-300          # kEpsilon of polishTheta / the FPKM denominators
DBL_MIN = 2.2250738585072014e-308
# walks of the sampler: parallel kernel with RSEM_B200_GIBBS_PF = 2 / 1 / 0, PF = 2 without the lean register-row draw,
# and the serial kernel
WALKS = ["2", "1", "0", "2-nofast", "serial"]
PARALLEL_WALKS = WALKS[:4]


def _set_walk(monkeypatch, walk, ctas=None):
    monkeypatch.setenv("RSEM_B200_TIMING", "1")
    monkeypatch.setenv("RSEM_B200_GIBBS", "serial" if walk == "serial" else "parallel")
    monkeypatch.setenv("RSEM_B200_GIBBS_PF", walk[0] if walk != "serial" else "2")
    if walk == "2-nofast":
        monkeypatch.setenv("RSEM_B200_GIBBS_FAST", "0")
    else:
        monkeypatch.delenv("RSEM_B200_GIBBS_FAST", raising=False)
    if ctas is None:
        monkeypatch.delenv("RSEM_B200_GIBBS_CTAS", raising=False)
    else:
        monkeypatch.setenv("RSEM_B200_GIBBS_CTAS", str(ctas))


def _timing(capfd):
    """(worker CTAs of chain 0, most passes of a chain) from the parallel path's timing lines; (None, None) if it did not run"""
    err = capfd.readouterr().err
    ctas = re.findall(r"gibbs chain 0 \((\d+) worker CTAs", err)
    passes = re.findall(r"most passes of a chain (\d+)", err)
    return (int(ctas[-1]) if ctas else None), (int(passes[-1]) if passes else None)


def _ofg_like(N, M, deg, seed, noise_scale):
    """rows of (sid, conprb) with the noise entry first (Gibbs.cpp:119-131); noise_scale moves the noise weight
    from negligible to dominant so that membership changes are rare / frequent"""
    rng = np.random.default_rng(seed)
    row_ptr, sid, conprb, ncpv = synth.random_matrix(N, M, deg, seed=seed, tiny_frac=0.0)
    conprb = np.where(conprb <= 0, 1e-30, conprb)
    rows_sid, rows_val, rp = [], [], [0]
    for i in range(N):
        a, b = int(row_ptr[i]), int(row_ptr[i + 1])
        s, v = list(np.abs(sid[a:b])), list(conprb[a:b])
        if rng.random() < 0.9:
            s.insert(0, 0)
            v.insert(0, float(np.median(conprb[a:b]) * noise_scale * rng.uniform(0.1, 10)))
        rows_sid += s
        rows_val += v
        rp.append(len(rows_sid))
    return np.array(rp, np.uint64), np.array(rows_sid, np.int32), np.array(rows_val, np.float64)


def _run_gpu(ctx, rp, sid, val, M, n0, init, alpha, totc, eel, mw, genes, burnin, gap, samples, seeds, upload=True):
    """-> count vectors, [sum_c, sum_c2, sum_tpm, sum_fpkm, sum_gene_c2], kernel launches of gibbs_run"""
    if upload:
        ctx.gibbs_upload(rp, sid, val, M)
    nc = len(samples)
    samples = np.ascontiguousarray(samples, np.int32)
    seeds = np.ascontiguousarray(seeds, np.uint32)
    init, genes = np.ascontiguousarray(init, np.int32), np.ascontiguousarray(genes, np.int32)
    alpha, eel, mw = (np.ascontiguousarray(x, np.float64) for x in (alpha, eel, mw))
    p = GibbsParams()
    p.M, p.burnin, p.gap, p.n_chains = M, burnin, gap, nc
    p.chain_samples = samples.ctypes.data_as(C.POINTER(C.c_int32))
    p.chain_seeds = seeds.ctypes.data_as(C.POINTER(C.c_uint32))
    p.n0, p.totc = n0, totc
    p.init_counts = init.ctypes.data_as(C.POINTER(C.c_int32))
    p.pseudo_counts = alpha.ctypes.data_as(C.POINTER(C.c_double))
    p.eel, p.mw = eel.ctypes.data_as(C.POINTER(C.c_double)), mw.ctypes.data_as(C.POINTER(C.c_double))
    p.n_genes = len(genes) - 1
    p.gene_start = genes.ctypes.data_as(C.POINTER(C.c_int32))
    total = int(samples.sum())
    cv = np.zeros((total, M + 1), np.int32)
    sums = [np.zeros(M + 1) for _ in range(4)] + [np.zeros(len(genes) - 1)]
    o = GibbsOut()
    o.count_vectors = cv.ctypes.data_as(C.POINTER(C.c_int32))
    o.sum_c, o.sum_c2, o.sum_tpm, o.sum_fpkm, o.sum_gene_c2 = (s.ctypes.data_as(C.POINTER(C.c_double)) for s in sums)
    before = ctx.launch_count()
    ctx.gibbs_run(p, o)
    return cv, sums, ctx.launch_count() - before


class Problem:
    """a matrix with the per-transcript inputs of a chain (defaults: no omitted transcript, alpha 0.7, mw 1)"""

    def __init__(self, rp, sid, val, M, seed=0, n0=100.0, alpha=None, init=None, eel=None, mw=None):
        rng = np.random.default_rng(seed)
        self.rp, self.sid, self.val, self.M, self.n0 = rp, sid, val, M, n0
        self.init = np.zeros(M + 1, np.int32) if init is None else np.asarray(init, np.int32)
        self.alpha = np.full(M + 1, 0.7) if alpha is None else np.asarray(alpha, np.float64)
        self.totc = float(self.alpha[self.init >= 0].sum()) + n0 + (len(rp) - 1)
        self.eel = np.concatenate([[0.0], rng.uniform(200, 2000, M)]) if eel is None else np.asarray(eel, np.float64)
        self.mw = np.ones(M + 1) if mw is None else np.asarray(mw, np.float64)
        self.genes = np.arange(1, M + 2, 3, dtype=np.int32)
        self.genes[-1] = M + 1


def _check(ctx, oracle, pb, samples, seeds, burnin, gap):
    """GPU vs oracle chain by chain: count vectors and the integer sums exact, TPM / FPKM sums to 1e-9"""
    cv, sums, launches = _run_gpu(ctx, pb.rp, pb.sid, pb.val, pb.M, pb.n0, pb.init, pb.alpha, pb.totc, pb.eel, pb.mw, pb.genes,
                                  burnin, gap, samples, seeds)
    at, ref_sums, ref_cv = 0, None, []
    for t, ns in enumerate(samples):
        cv_ref, s = oracle.gibbs_chain(pb.rp, pb.sid, pb.val, pb.M, pb.n0, pb.init, pb.alpha, pb.totc, pb.eel, pb.mw, pb.genes,
                                       burnin, gap, ns, int(seeds[t]))
        assert np.array_equal(cv[at:at + ns], cv_ref), f"chain {t} differs"
        at += ns
        ref_cv.append(cv_ref)
        ref_sums = s if ref_sums is None else [x + y for x, y in zip(ref_sums, s)]
    for k, name in ((0, "sum_c"), (1, "sum_c2"), (4, "sum_gene_c2")):
        assert np.array_equal(sums[k], ref_sums[k]), name
    for k, name in ((2, "sum_tpm"), (3, "sum_fpkm")):
        assert np.allclose(sums[k], ref_sums[k], rtol=1e-9, atol=0.0), name
    return cv, ref_sums, launches


# ---- what a matrix looks like (the edge a case is about) ----------------------------------------------------------------
def _rows(rp):
    return np.diff(np.asarray(rp, np.int64))


def _components(rp, sid, M):
    """connected components of the read x transcript graph, transcript 0 excluded ->
    (transcripts in the component of each read (0: only the noise entry), component label of transcripts 0..M)"""
    N = len(rp) - 1
    rows = np.repeat(np.arange(N), _rows(rp))
    m = sid != 0
    n = N + M + 1
    g = sparse.coo_matrix((np.ones(int(m.sum())), (rows[m], N + sid[m].astype(np.int64))), shape=(n, n))
    _, lab = csgraph.connected_components(g, directed=False)
    ntr = np.bincount(lab[N + 1:], minlength=lab.max() + 1)
    has = np.zeros(N, bool)
    has[rows[m]] = True
    return np.where(has, ntr[lab[:N]], 0), lab[N:]


def _row_ids(rp, sid, i):
    return sid[int(rp[i]):int(rp[i + 1])]


def _csr(rows):
    """list of (ids, values) -> row_ptr, sid, conprb"""
    rp = np.zeros(len(rows) + 1, np.uint64)
    rp[1:] = np.cumsum([len(r[0]) for r in rows])
    sid = np.concatenate([np.asarray(r[0], np.int32) for r in rows]) if rows else np.zeros(0, np.int32)
    val = np.concatenate([np.asarray(r[1], np.float64) for r in rows]) if rows else np.zeros(0)
    return rp, sid.astype(np.int32), val


def _to_rows(rp, sid, val):
    return [(list(sid[int(rp[i]):int(rp[i + 1])]), list(val[int(rp[i]):int(rp[i + 1])])) for i in range(len(rp) - 1)]


# ---- the original two tests ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["parallel", "serial"])
@pytest.mark.parametrize("noise_scale,seed", [(1e-30, 3), (1.0, 10), (30.0, 213)])
def test_chains_match_oracle(ctx, oracle, mode, noise_scale, seed, monkeypatch):
    N, M = 3000, 150
    rp, sid, val = _ofg_like(N, M, 4, seed=seed, noise_scale=noise_scale)
    n0 = 40.0
    init = np.zeros(M + 1, np.int32)
    init[[5, 77]] = -1                                   # omitted transcripts never appear in a row
    keep = ~np.isin(sid, [5, 77])
    # drop omitted ids from the rows
    new_rp = [0]
    for i in range(N):
        new_rp.append(new_rp[-1] + int(keep[int(rp[i]):int(rp[i + 1])].sum()))
    rp, sid, val = np.array(new_rp, np.uint64), sid[keep], val[keep]
    if np.any(np.diff(rp.astype(np.int64)) == 0):
        pytest.skip("generator produced an empty row")
    alpha = np.full(M + 1, 0.7)
    totc = (M + 1 - 2) * 0.7 + n0 + N
    rng = np.random.default_rng(1)
    eel = np.concatenate([[0.0], rng.uniform(200, 2000, M)])
    mw = np.ones(M + 1)
    genes = np.arange(1, M + 2, 3, dtype=np.int32)
    genes[-1] = M + 1
    samples, burnin, gap = [3, 2, 2], 6, 2
    seeds = oracle.chain_seeds(2024, 3)
    monkeypatch.setenv("RSEM_B200_GIBBS", mode)
    cv, sums, _ = _run_gpu(ctx, rp, sid, val, M, n0, init, alpha, totc, eel, mw, genes, burnin, gap, samples, seeds)
    at, ref_sums = 0, None
    for t, ns in enumerate(samples):
        cv_ref, s = oracle.gibbs_chain(rp, sid, val, M, n0, init, alpha, totc, eel, mw, genes, burnin, gap, ns, int(seeds[t]))
        assert np.array_equal(cv[at:at + ns], cv_ref), f"chain {t} differs"
        at += ns
        ref_sums = s if ref_sums is None else [x + y for x, y in zip(ref_sums, s)]
    for got, ref in zip(sums, ref_sums):
        assert np.allclose(got, ref, rtol=1e-9, atol=1e-9)
    # the noise count really moves in the stressed cases (otherwise the roll-back path is not exercised)
    if noise_scale >= 1.0:
        assert len(set(cv[:, 0].tolist())) > 1


def _family_matrix(N, M, seed, max_family, junk):
    """disjoint isoform families (one connected component each; <= 31 transcripts: register-resident counts, more: counts
    in L2), reads hit a run of members of one family, the noise entry first; a few rows longer than 16 entries"""
    rng = np.random.default_rng(seed)
    sizes, tot = [], 0
    while tot < M:
        k = min(int(rng.integers(1, max_family + 1)), M - tot)
        sizes.append(k)
        tot += k
    sizes = np.array(sizes)
    start = np.concatenate([[1], 1 + np.cumsum(sizes)[:-1]])
    wgt = rng.random(len(sizes)) ** 3 + 1e-3
    fam = rng.choice(len(sizes), size=N, p=wgt / wgt.sum())
    rows_sid, rows_val, rp = [], [], [0]
    for i in range(N):
        k = int(sizes[fam[i]])
        d = k if rng.random() < 0.7 else int(rng.integers(1, k + 1))
        first = int(start[fam[i]]) + int(rng.integers(0, k - d + 1))
        s = [0] + list(range(first, first + d))
        v = list(10.0 ** rng.uniform(-12, -3, d))
        nz = 10.0 ** rng.uniform(-14, -5, 1)[0] if rng.random() < junk else 10.0 ** rng.uniform(-60, -40, 1)[0]
        if rng.random() < 0.05:   # a row without a noise entry
            s, v = s[1:], v
        else:
            v = [nz] + v
        rows_sid += s
        rows_val += v
        rp.append(len(rows_sid))
    return np.array(rp, np.uint64), np.array(rows_sid, np.int32), np.array(rows_val, np.float64)


@pytest.mark.parametrize("pf", WALKS)
@pytest.mark.parametrize("max_family,junk,prior", [pytest.param(12, 0.02, False, id="12-0.02"),
                                                   pytest.param(40, 0.3, False, id="40-0.3"),
                                                   pytest.param(12, 0.02, True, id="12-0.02-prior"),
                                                   pytest.param(40, 0.3, True, id="40-0.3-prior")])
def test_family_components_match_oracle(ctx, oracle, pf, max_family, junk, prior, monkeypatch, capfd):
    """the component walk of the parallel sampler (RSEM_B200_GIBBS_PF = 2 pipelined + converged, 1 pipelined per segment, 0
    row-at-a-time; PF = 2 without the lean register-row draw; the serial kernel) on the matrix shape it is built for: many
    components of very different sizes, segments of hundreds of rows (many 16-slot batches), rows that fill a lane group
    exactly and rows longer than one.  `prior`: a --prior-like pseudo-count per transcript (register-resident components
    read it through their local ids)"""
    N, M = 30000, 1500
    rp, sid, val = _family_matrix(N, M, seed=max_family, max_family=max_family, junk=junk)
    rng = np.random.default_rng(2)
    alpha = np.random.default_rng(3).uniform(0.1, 3.0, M + 1) if prior else np.ones(M + 1)
    pb = Problem(rp, sid, val, M, n0=1500.0, alpha=alpha, eel=np.concatenate([[0.0], rng.uniform(200, 2000, M)]))
    pb.genes = np.arange(1, M + 2, 4, dtype=np.int32)
    pb.genes[-1] = M + 1
    _set_walk(monkeypatch, pf)
    cv, _, _ = _check(ctx, oracle, pb, [2, 2], oracle.chain_seeds(7, 2), 3, 1)
    assert len(set(cv[:, 0].tolist())) > 1   # reads do move in and out of the noise transcript
    lens = _rows(rp)
    assert lens.max() > 16 or max_family <= 12
    ntr, _ = _components(rp, sid, M)
    assert ntr.max() < 32 or max_family > 31   # both kinds of component when families can exceed 31 transcripts
    if max_family > 31:
        assert (ntr >= 32).any() and ((ntr > 0) & (ntr < 32)).any()
    if prior:   # distinct pseudo-counts inside register-resident components
        assert len(np.unique(alpha[sid[sid > 0]])) > 100
    assert (_timing(capfd)[0] is None) == (pf == "serial")


# ---- 1. dispatch boundary and the generator's 624-word blocks ----------------------------------------------------------------
@pytest.mark.parametrize("walk", WALKS)
@pytest.mark.parametrize("N1", [1247, 1248, 1249, 1871, 1872, 1873, 2497])
def test_dispatch_boundary_match_oracle(ctx, oracle, walk, N1, monkeypatch, capfd):
    """N1 < 1248 runs the serial kernel whatever the walk; from 1248 on the parallel one, whose generator CTA hands out the
    stream in 624-word blocks: sweeps that end exactly on a block (1248, 1872), one past it, and more than four blocks"""
    M = 150
    rp, sid, val = _ofg_like(N1, M, 4, seed=N1, noise_scale=1.0)
    assert len(rp) - 1 == N1
    _set_walk(monkeypatch, walk)
    _, _, launches = _check(ctx, oracle, Problem(rp, sid, val, M, seed=N1, n0=40.0), [1, 3, 2], oracle.chain_seeds(N1, 3), 2, 2)
    ctas, _ = _timing(capfd)
    parallel = walk != "serial" and N1 >= 1248
    assert (ctas is not None) == parallel
    assert launches == 1   # 3 chains: one wave on the parallel path, one serial launch otherwise


# ---- 2. launch waves ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("walk", WALKS)
def test_waves_match_oracle(ctx, oracle, walk, monkeypatch, capfd, record_property):
    """600 chains of 1 or 2 samples: a wave holds at most half the co-resident CTAs' worth of chains (<= 528 on an H100), so
    the parallel path needs several cooperative launches; every chain's vectors land at its own offset"""
    N1, M, nc = 1250, 150, 600
    rp, sid, val = _ofg_like(N1, M, 4, seed=600, noise_scale=1.0)
    samples = np.random.default_rng(600).integers(1, 3, nc)
    seeds = oracle.chain_seeds(600, nc)
    seeds[0], seeds[nc // 2] = 0, 0xFFFFFFFF
    assert len(set(samples.tolist())) == 2
    _set_walk(monkeypatch, walk)
    _, _, launches = _check(ctx, oracle, Problem(rp, sid, val, M, seed=600, n0=40.0), samples, seeds, 1, 1)
    ctas, _ = _timing(capfd)
    if walk == "serial":
        assert launches == 1 and ctas is None
    else:
        assert ctas is not None and launches >= 2
        record_property("waves", launches)
        record_property("worker_ctas", ctas)


# ---- 3. worker CTAs per chain -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("walk", PARALLEL_WALKS)
@pytest.mark.parametrize("n_ctas", [1, 2, 64, 512])
def test_worker_ctas_match_oracle(ctx, oracle, walk, n_ctas, monkeypatch, capfd, record_property):
    """the flip bitmaps (W = 41 words at N1 = 1300) split into per-CTA slices: one slice, two, more CTAs than words (empty
    slices), and as many as the residency cap allows; noise-heavy rows so that flips land in many slices"""
    N1, M = 1300, 150
    W = (N1 + 31) // 32
    rp, sid, val = _ofg_like(N1, M, 4, seed=64, noise_scale=30.0)
    _set_walk(monkeypatch, walk, ctas=n_ctas)
    cv, _, launches = _check(ctx, oracle, Problem(rp, sid, val, M, seed=64, n0=40.0), [2, 3], oracle.chain_seeds(64, 2), 2, 1)
    ctas, _ = _timing(capfd)
    assert launches == 1
    if n_ctas < 512:
        assert ctas == n_ctas
    else:   # the residency cap may lower the request
        assert W < ctas <= 512
    record_property("worker_ctas", ctas)
    assert len(set(cv[:, 0].tolist())) > 1


# ---- 4 + 6. row lengths against the lane group; per-transcript pseudo-counts ------------------------------------------------------
LANE_LENS = (15, 16, 17, 31, 32, 33, 48)


def _lane_matrix(N, seed):
    """families of exactly 30 and 31 (counts in registers) and 32 and 33 transcripts (counts in L2) plus small ones; rows of
    15, 16, 17, 31, 32, 33 and 48 entries drawn from one family, with repeated ids (a read with two alignments to one
    transcript) - the only way a row of a register-resident family gets longer than 32 entries; rows of <= 16 entries made
    of two alternating ids, so that the read's previous and its new assignment both sit in several lanes"""
    rng = np.random.default_rng(seed)
    sizes = [30, 31, 32, 33, 1, 5, 16, 17]
    start = 1 + np.concatenate([[0], np.cumsum(sizes)[:-1]])
    fams = [np.arange(s, s + k) for s, k in zip(start, sizes)]

    def row(ids, noise):
        v = list(10.0 ** rng.uniform(-6, -2, len(ids)))
        return ([0] + list(ids), [10.0 ** rng.uniform(-6, -2)] + v) if noise else (list(ids), v)

    rows = []
    for f in fams:
        rows.append(row(rng.permutation(f), True))   # one row over the whole family keeps it one component
        if len(f) > 1:
            a, b = rng.choice(f, 2, replace=False)
            for L in (15, 16, 6):
                rows.append(row(([a, b] * 8)[:L], False))
    while len(rows) < N:
        f = fams[int(rng.integers(len(fams)))]
        L = int(rng.choice(LANE_LENS))
        noise = rng.random() < 0.8
        n = L - int(noise)
        rows.append(row(rng.choice(f, n, replace=n > len(f) or rng.random() < 0.5), noise))
    rows = [rows[i] for i in rng.permutation(len(rows))]
    return _csr(rows) + (int(sum(sizes)),)


@pytest.mark.parametrize("walk", WALKS)
@pytest.mark.parametrize("prior", [False, True])
def test_lane_group_rows_match_oracle(ctx, oracle, walk, prior, monkeypatch):
    rp, sid, val, M = _lane_matrix(2500, seed=17)
    lens = _rows(rp)
    ntr, _ = _components(rp, sid, M)
    assert {30, 31, 32, 33} <= set(ntr.tolist())
    assert set(LANE_LENS) <= set(lens.tolist())
    rep = np.array([len(set(_row_ids(rp, sid, i).tolist())) < lens[i] for i in range(len(lens))])
    reg = (ntr > 0) & (ntr < 32)
    assert (rep & reg & (lens > 32)).any() and (rep & (ntr >= 32)).any()
    for kind in (reg, ntr >= 32):   # every id of the row repeated: whatever the previous and the new assignment are
        assert any(lens[i] <= 16 and np.unique(_row_ids(rp, sid, i), return_counts=True)[1].min() >= 2 for i in np.flatnonzero(kind))
    alpha = np.random.default_rng(5).uniform(0.1, 3.0, M + 1) if prior else None
    _set_walk(monkeypatch, walk)
    cv, _, _ = _check(ctx, oracle, Problem(rp, sid, val, M, seed=4, n0=200.0, alpha=alpha), [2, 1, 3],
                      oracle.chain_seeds(44, 3), 3, 1)
    assert len(set(cv[:, 0].tolist())) > 1


# ---- 5. rows longer than the serial kernel's shared-memory array -------------------------------------------------------------------
@pytest.mark.parametrize("walk", WALKS)
def test_long_rows_match_oracle(ctx, oracle, walk, monkeypatch):
    """rows of 2047, 2048, 2049 and 5000 entries (repeated ids) in a register-resident family and in an L2 component"""
    rng = np.random.default_rng(2048)
    base, reg = 200, np.arange(201, 221)
    rows = _to_rows(*_ofg_like(1296, base, 4, seed=2048, noise_scale=1.0))
    rows.append(([0] + list(reg), list(10.0 ** rng.uniform(-6, -2, 21))))
    for _ in range(40):
        ids = list(rng.choice(reg, int(rng.integers(1, 12))))
        rows.append(([0] + ids, list(10.0 ** rng.uniform(-6, -2, len(ids) + 1))))
    for L, pool in ((2047, reg), (5000, reg), (2048, np.arange(1, base + 1)), (2049, np.arange(1, base + 1))):
        rows.append(([0] + list(rng.choice(pool, L - 1)), list(10.0 ** rng.uniform(-6, -2, L))))
    rows = [rows[i] for i in rng.permutation(len(rows))]
    rp, sid, val = _csr(rows)
    M = 220
    lens = _rows(rp)
    ntr, _ = _components(rp, sid, M)
    assert {2047, 2048, 2049, 5000} <= set(lens.tolist())
    assert ((lens > 2048) & (ntr > 0) & (ntr < 32)).any() and ((lens > 2048) & (ntr >= 32)).any()
    _set_walk(monkeypatch, walk)
    _check(ctx, oracle, Problem(rp, sid, val, M, seed=5, n0=100.0), [2, 2], oracle.chain_seeds(2048, 2), 2, 1)


# ---- 7. per-sample edges: mw / eel below epsilon, omitted transcripts ------------------------------------------------------------------
def _with_omitted(seed, n_omit):
    """family matrix whose register-resident families have holes: omitted transcripts (init = -1) taken out of every row (a
    row left without entries keeps a lone noise entry)"""
    N, M = 3000, 300
    rp, sid, val = _family_matrix(N, M, seed=seed, max_family=12, junk=0.3)
    _, lab = _components(rp, sid, M)
    inner = [t for t in range(2, M) if lab[t - 1] == lab[t] == lab[t + 1]]
    omitted = np.random.default_rng(seed).choice(inner, n_omit, replace=False)
    gone = set(omitted.tolist())
    rows = []
    for ids, v in _to_rows(rp, sid, val):
        keep = [k for k, t in enumerate(ids) if t not in gone]
        rows.append(([ids[k] for k in keep], [v[k] for k in keep]) if keep else ([0], [1e-8]))
    rp, sid, val = _csr(rows)
    init = np.zeros(M + 1, np.int32)
    init[omitted] = -1
    ntr, lab = _components(rp, sid, M)
    assert ntr.max() < 32 and not np.isin(sid, omitted).any()
    # most omitted ids sit between two transcripts of one (register-resident) component: its local ids skip them
    present = np.unique(sid[sid > 0])
    inside = [lab[present[present < t].max()] == lab[present[present > t].min()] for t in omitted]
    assert sum(inside) >= n_omit // 2
    return rp, sid, val, M, init


def _fpkm_denominator(counts, alpha, totc, mw, eel, zero_eel):
    """polishTheta + the FPKM denominator of one sample, with or without zeroing transcripts whose eel is below epsilon"""
    th = np.where(counts < 0, 0.0, (counts + alpha) / totc)
    drop = (mw < EPS) | ((eel < EPS) if zero_eel else False)
    drop[0] = False
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        th = np.where(drop, 0.0, th / mw)
    th = th / th.sum()
    return th[1:][eel[1:] >= EPS].sum()


@pytest.mark.parametrize("walk", WALKS)
@pytest.mark.parametrize("edge", ["weights", "no_eel"])
def test_per_sample_edges_match_oracle(ctx, oracle, walk, edge, monkeypatch):
    """weights: transcripts with mw below epsilon, and transcripts with eel below epsilon whose mw is exactly epsilon - their
    theta / mw outweighs the rest by more than 1 / epsilon, so unless they are zeroed the FPKM denominator falls below
    epsilon and is replaced by 1; no_eel: every eel below epsilon (both denominators fall back to 1, TPM and FPKM are 0)"""
    rp, sid, val, M, init = _with_omitted(77, 12)
    rng = np.random.default_rng(78)
    alive = np.flatnonzero(init[1:] >= 0) + 1
    if edge == "weights":
        pick = rng.choice(alive, 20, replace=False)
        small_mw, small_eel = pick[:10], pick[10:]
        mw = np.concatenate([[1.0], 10.0 ** rng.uniform(3, 4, M)])
        eel = np.concatenate([[0.0], rng.uniform(200, 2000, M)])
        mw[small_mw] = np.array([1e-305, 0.0, 5e-324, 1e-301, 0.0] * 2)
        eel[small_eel] = np.array([0.0, 1e-305, 5e-324, 1e-301, -0.0] * 2)
        mw[small_eel] = EPS
    else:
        mw = np.ones(M + 1)
        eel = np.where(rng.random(M + 1) < 0.5, 0.0, 1e-301)
    pb = Problem(rp, sid, val, M, n0=300.0, init=init, eel=eel, mw=mw)
    samples = [2, 3]
    _set_walk(monkeypatch, walk)
    cv, ref_sums, _ = _check(ctx, oracle, pb, samples, oracle.chain_seeds(77, 2), 2, 1)
    assert (cv[:, init < 0] == -1).all()
    if edge == "weights":   # the eel half of the zeroing decides every sample
        for c in cv:
            assert _fpkm_denominator(c, pb.alpha, pb.totc, mw, eel, True) > 1e-6
            assert _fpkm_denominator(c, pb.alpha, pb.totc, mw, eel, False) < EPS
    else:
        assert not ref_sums[2].any() and not ref_sums[3].any()


# ---- 8. row contents: noise-only rows, subnormal products ------------------------------------------------------------------------
@pytest.mark.parametrize("walk", WALKS)
def test_row_contents_match_oracle(ctx, oracle, walk, monkeypatch):
    N, M, n0 = 3000, 400, 100.0
    rng = np.random.default_rng(8)
    rows = _to_rows(*_family_matrix(N, M, seed=8, max_family=12, junk=0.3))
    alpha = rng.uniform(0.1, 3.0, M + 1)
    for i in rng.choice(len(rows), len(rows) // 8, replace=False):   # every product of the row subnormal, none zero
        rows[i] = (rows[i][0], list(10.0 ** rng.uniform(-320, -312, len(rows[i][0]))))
    for i in sorted(rng.choice(len(rows), 150, replace=False), reverse=True):   # reads with only the noise entry
        rows.insert(int(i), ([0], [float(10.0 ** rng.uniform(-8, -3))]))
    rp, sid, val = _csr(rows)
    lens = _rows(rp)
    ntr, _ = _components(rp, sid, M)
    assert ((ntr == 0) & (lens == 1)).sum() >= 150
    sub = np.array([val[int(rp[i]):int(rp[i + 1])].max() * (len(rp) - 1 + n0 + alpha.max()) < DBL_MIN for i in range(len(lens))])
    assert sub.sum() >= len(lens) // 10 and val.min() * alpha.min() > 0.0
    _set_walk(monkeypatch, walk)
    _check(ctx, oracle, Problem(rp, sid, val, M, seed=8, n0=n0, alpha=alpha), [2, 2], oracle.chain_seeds(8, 2), 2, 1)


# ---- 9. chain shapes --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("walk", WALKS)
def test_chain_shapes_match_oracle(ctx, oracle, walk, monkeypatch):
    """no burn-in, chains of 1 sample next to chains of 4, a gap of 3"""
    rp, sid, val = _family_matrix(2000, 200, seed=9, max_family=40, junk=0.3)
    _set_walk(monkeypatch, walk)
    _check(ctx, oracle, Problem(rp, sid, val, 200, seed=9, n0=100.0), [1, 4, 1, 4], oracle.chain_seeds(9, 4), 0, 3)


@pytest.mark.parametrize("walk", ["2", "serial"])
def test_no_reads_match_oracle(ctx, oracle, walk, monkeypatch):
    """N1 = 0: every sample is the initial counts (init + n0 on the noise transcript)"""
    M = 5
    init = np.array([0, 0, -1, 0, 0, 0], np.int32)
    pb = Problem(np.zeros(1, np.uint64), np.zeros(0, np.int32), np.zeros(0), M, n0=7.0, init=init)
    _set_walk(monkeypatch, walk)
    cv, _, _ = _check(ctx, oracle, pb, [2, 1], oracle.chain_seeds(1, 2), 0, 2)
    assert (cv == init + np.array([7, 0, 0, 0, 0, 0])).all()


# ---- 10. many passes of the fixed-point iteration ----------------------------------------------------------------------------------
@pytest.mark.parametrize("walk", PARALLEL_WALKS)
def test_many_passes_match_oracle(ctx, oracle, walk, monkeypatch, capfd, record_property):
    """a small noise count and noise entries as heavy as the rest: reads join and leave the noise transcript so often that a
    sweep needs more than two passes - the restart from the sweep's copy of the counts runs again and again"""
    rp, sid, val = _ofg_like(3000, 150, 4, seed=11, noise_scale=1.0)
    samples, burnin, gap = [2, 2], 4, 1
    _set_walk(monkeypatch, walk)
    _check(ctx, oracle, Problem(rp, sid, val, 150, seed=11, n0=5.0), samples, oracle.chain_seeds(11, 2), burnin, gap)
    _, passes = _timing(capfd)
    sweeps = burnin + 1 + (max(samples) - 1) * gap   # sweeps with live counts of every chain
    record_property("passes_per_sweep", passes / sweeps)
    assert passes > 2 * sweeps


# ---- a row without entries ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N1", [1000, 3000])
def test_empty_row_refused_before_launch(ctx, oracle, N1, monkeypatch):
    """both paths refuse a read without entries with the same message and launch nothing; the context stays usable"""
    M = 150
    rp, sid, val = _ofg_like(N1, M, 4, seed=N1, noise_scale=1.0)
    rows = _to_rows(rp, sid, val)
    rows[N1 // 2] = ([], [])
    erp, esid, eval_ = _csr(rows)
    pb = Problem(erp, esid, eval_, M, n0=40.0)
    msgs = []
    for walk in ("2", "serial"):
        _set_walk(monkeypatch, walk)
        ctx.gibbs_upload(erp, esid, eval_, M)
        before = ctx.launch_count()
        with pytest.raises(RsemB200Error) as e:
            _run_gpu(ctx, erp, esid, eval_, M, pb.n0, pb.init, pb.alpha, pb.totc, pb.eel, pb.mw, pb.genes, 1, 1, [1], [3],
                     upload=False)
        assert ctx.launch_count() == before
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1] and "a read without any entry" in msgs[0]
    _set_walk(monkeypatch, "2")
    _check(ctx, oracle, Problem(rp, sid, val, M, n0=40.0), [2, 1], oracle.chain_seeds(N1, 2), 1, 1)


@pytest.fixture(scope="module")
def ctx(built):
    import rsem_b200
    c = rsem_b200.Context(0)
    yield c
    c.close()
