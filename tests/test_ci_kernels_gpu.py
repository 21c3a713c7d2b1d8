"""K8, Phase II of rsem-calculate-credibility-intervals (ci_kernels.cu), through the C ABI against the CPU restatement
ro_ci_phase2 (oracle/rsem_oracle.c), bit for bit.

Every case pushes a sample-major matrix through ci_begin / ci_push / ci_end and compares the transcript, gene and
isoform outputs with the restatement as uint32 bits, then checks from CiStats and the block rule (ci_phase2.py) that
the run reached the edge it names.  Inputs stay in the domain Phase I produces: finite, non-negative TPMs (+0.0 and
positive subnormals included: tiny Gamma draws underflow) and positive normal l_bars."""
import ctypes
import os
import threading

import numpy as np
import pytest

import ci_phase2 as cp
from rsem_b200.capi import CiParams, RsemB200Error, _p

pytestmark = pytest.mark.gpu

F32 = np.float32
FLT_MIN = np.finfo(F32).tiny
STAGE_BYTES = 32 << 20  # ci_push's pinned stage
C_INT = ctypes.c_int32


@pytest.fixture(scope="module")
def ctx(built):
    import rsem_b200
    with rsem_b200.Context(0) as c:
        yield c


def _params(gene_start, n, threshold, budget=0, isoform_start=None, parts=None):
    """-> (CiParams, the arrays it points into)"""
    gs = np.ascontiguousarray(gene_start, np.int32)
    pg = np.ascontiguousarray([0, len(gs) - 1] if parts is None else parts, np.int32)
    iso = None if isoform_start is None else np.ascontiguousarray(isoform_start, np.int32)
    p = CiParams(M=int(gs[-1] - 1), n_genes=len(gs) - 1, gene_start=_p(gs, C_INT),
                 n_isoforms=0 if iso is None else len(iso) - 1, n_parts=len(pg) - 1, isoform_start=_p(iso, C_INT),
                 part_gene_start=_p(pg, C_INT), n_samples=n, threshold=threshold, device_budget=budget)
    return p, (gs, pg, iso)


def _push_chunks(ctx, tm, l_bars, chunk=4096):
    n = tm.shape[1]
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        ctx.ci_push(np.ascontiguousarray(tm[:, a:b].T), l_bars[a:b], a)


def _gpu(ctx, tm, l_bars, gene_start, threshold, budget=0, isoform_start=None, parts=None, push=None):
    """tm: M x n transcript-major TPMs, pushed as sample-major rows -> (transcripts, genes, isoforms, CiStats)"""
    M, n = tm.shape
    params, keep = _params(gene_start, n, threshold, budget, isoform_start, parts)
    ctx.ci_begin(params)
    (push or _push_chunks)(ctx, tm, l_bars)
    return ctx.ci_end(M, len(gene_start) - 1, 0 if isoform_start is None else len(isoform_start) - 1)


def _same_bits(got, want, what):
    g, w = got.view(np.uint32), want.view(np.uint32)
    bad = np.argwhere(g != w)
    assert bad.size == 0, (f"{what}: {len(bad)} floats differ, first at {tuple(bad[0])}: "
                           f"{got[tuple(bad[0])]!r} vs {want[tuple(bad[0])]!r}")


def _check(ctx, oracle, tm, l_bars, gene_start, threshold, budget=0, isoform_start=None, parts=None, push=None):
    """-> (CiStats, the restatement's outputs)"""
    tr, ge, iso, st = _gpu(ctx, tm, l_bars, gene_start, threshold, budget, isoform_start, parts, push)
    want = oracle.ci_phase2(tm, l_bars, gene_start, threshold, isoform_start=isoform_start, part_gene_start=parts)
    for got, w, what in zip((tr, ge, iso), want, ("transcripts", "genes", "isoforms")):
        _same_bits(got, w, what)
    return st, want


def _l_bars(rng, n):
    return np.exp(rng.uniform(np.log(30.0), np.log(1e4), n)).astype(F32)


def _gene_start(sizes):
    return np.concatenate([[1], 1 + np.cumsum(sizes)]).astype(np.int64).tolist()


@pytest.mark.parametrize("n", range(1, 10))
def test_every_threshold_small_n(ctx, oracle, n):
    """n = 1 .. 9: Tukey's hinges for residues 0 - 3 with quotient 0 and 1, and the interval search at every
    threshold 0 .. n - 1"""
    rng = np.random.default_rng(100 + n)
    gene_start = _gene_start([1, 2, 3, 4, 1, 5])
    M = gene_start[-1] - 1
    tm = rng.gamma(0.7, 3.0, (M, n)).astype(F32)
    tm[::3] = rng.integers(0, 3, (len(tm[::3]), n)).astype(F32) * F32(0.5)  # ties
    l_bars = _l_bars(rng, n)
    for threshold in range(n):
        _check(ctx, oracle, tm, l_bars, gene_start, threshold)


def _tie_rows(rng, n):
    sub = lambda k: rng.integers(1, 1 << 23, k).astype(np.uint32).view(F32)  # positive subnormals
    rows = [
        rng.choice(F32([0.5, 1.0, 2.0]), n),                              # three levels
        rng.choice(F32([0.0, 0.25, 0.75, 3.0]), n),                       # four levels with zero
        np.full(n, F32(3.0)),                                             # constant: cqv = 0
        np.zeros(n, F32),                                                 # all zero
        np.where(rng.random(n) < 0.5, F32(0), sub(n)),                    # zeros and subnormals
        rng.choice(np.concatenate([F32([0, FLT_MIN]), sub(2)]), n),       # zeros, FLT_MIN and its neighbours below
        rng.choice(F32([np.nextafter(F32(1), F32(0)), 1.0, np.nextafter(F32(1), F32(2))]), n),  # 1 ulp apart
    ]
    # runs of ties across the threshold at the bottom and the top: k1 low, k2 high, the middle one value
    t = cp.threshold(0.95, n)
    for k1, k2 in ((t, t), (t + 1, t - 1 if t else 0), (t // 2, t + 2), (0, t + 1)):
        k1, k2 = min(k1, n), min(k2, max(0, n - k1))
        r = np.full(n, F32(2.0))
        r[:k1], r[n - k2:] = F32(1.0), F32(5.0)
        rows.append(rng.permutation(r))
    rows.append(rng.gamma(0.5, 1.0, n).astype(F32))
    return np.stack(rows).astype(F32)


@pytest.mark.parametrize("n", [40, 41, 42, 43, 1001])
def test_ties_zeros_subnormals(ctx, oracle, n):
    """quantised, constant and all-zero rows, zeros with subnormals and FLT_MIN, neighbours one ulp apart, and tie runs
    straddling the threshold on both pointers; genes sum them (subnormal sums stay exact, 1-ulp sums round)"""
    rng = np.random.default_rng(n)
    tm = _tie_rows(rng, n)
    M = len(tm)
    gene_start = _gene_start([2, 1, 3, 1, 2, M - 9])
    l_bars = _l_bars(rng, n)
    for threshold in sorted({0, cp.threshold(0.95, n), cp.threshold(0.5, n), n - 1}):
        st, (tr, ge, _) = _check(ctx, oracle, tm, l_bars, gene_start, threshold)
        assert (tr[:, 2] == 0).any() and (tr[:, 2] > 0).any()  # both cqv branches


def test_gene_sum_order(ctx, oracle):
    """a gene of 2^24 then many 1.0s and the same transcripts reversed: float sums in transcript order round the
    ones away in the first and keep them in the second"""
    rng = np.random.default_rng(24)
    n, k = 1000, 15
    big = (F32(2**24) + 2 * rng.integers(0, 1000, n)).astype(F32)
    ones = np.ones((k, n), F32)
    tm = np.concatenate([big[None], ones, ones, big[None], rng.gamma(1.0, 1.0, (3, n)).astype(F32)])
    gene_start = _gene_start([k + 1, k + 1, 3])
    st, (tr, ge, _) = _check(ctx, oracle, tm, _l_bars(rng, n), gene_start, cp.threshold(0.95, n))
    assert not np.array_equal(ge[0].view(np.uint32), ge[1].view(np.uint32))


def test_fpkm_rounding(ctx, oracle):
    """l_bar spread over [30, 10 000]: FPKM = (float)(1e3 / (double)l_bar * tpm); the float evaluation of the same
    expression differs in the last bit for many of these inputs"""
    rng = np.random.default_rng(338)
    n, sizes = 2000, rng.integers(1, 6, 60)
    gene_start = _gene_start(sizes)
    M = gene_start[-1] - 1
    tm = rng.gamma(0.6, 20.0, (M, n)).astype(F32)
    l_bars = _l_bars(rng, n)
    exact = (1e3 / l_bars.astype(np.float64) * tm.astype(np.float64)).astype(F32)
    in_float = F32(1e3) / l_bars * tm
    assert (exact != in_float).mean() > 0.05
    _check(ctx, oracle, tm, l_bars, gene_start, cp.threshold(0.95, n))


def test_default_scale(ctx, oracle):
    """the driver's default nCV 1000 x nSpC 50 = 50 000 samples over 24 000 transcripts in 9 000 genes with the default
    budget: the first block stops at INT32_MAX // n rows, so one segmented sort of about 2.147e9 keys"""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 30e9:
        pytest.skip(f"{free / 1e9:.1f} GB of device memory free; the default-scale case needs about 30 GB")
    rng = np.random.default_rng(50000)
    n, m = 50_000, 9_000
    sizes = np.ones(m, np.int64)
    extra = rng.choice(np.repeat(np.arange(m), 8), 15_000, replace=False)
    np.add.at(sizes, extra, 1)
    gene_start = _gene_start(sizes)
    M = gene_start[-1] - 1
    assert M == 24_000
    tm = np.empty((M, n), F32)
    for a in range(0, M, 2000):
        tm[a:a + 2000] = rng.standard_exponential((min(2000, M - a), n), dtype=F32) ** 3 * F32(40)
    l_bars = _l_bars(rng, n)
    thr = cp.threshold(0.95, n)
    st, _ = _check(ctx, oracle, tm, l_bars, gene_start, thr)
    budget = free - (512 << 20)  # ci_begin's default, give or take what this process allocated since
    resident, rows_cap, max_rows, all_rows = cp.block_rule(gene_start, n, budget)
    assert resident and st.resident == 1
    assert rows_cap == cp.INT32_MAX // n == 42_949
    blocks = cp.blocks(gene_start, rows_cap)
    assert st.blocks == len(blocks) >= 2
    assert blocks[0] >= rows_cap - max_rows
    print(f"\ndefault scale: n = {n}, M = {M}, {m} genes, {all_rows} rows in {st.blocks} blocks {blocks}; "
          f"largest segmented sort {blocks[0] * n} keys (INT32_MAX - {cp.INT32_MAX - blocks[0] * n}); "
          f"device ms: transpose {st.transpose_ms:.0f}, sums {st.sums_ms:.0f}, sort {st.sort_ms:.0f}, "
          f"intervals {st.interval_ms:.0f}")


def test_rows_wider_than_the_stage(ctx, oracle):
    """M = 8 388 609 in 2-transcript genes, n = 3: a row larger than the 32 MiB stage (the pageable push path), about
    4.2 M multi-transcript genes in one block (the gene sums stride over grid.y) and w / 32 > 65 535 (so does the
    transpose)"""
    rng = np.random.default_rng(8388609)
    M, n = 8_388_609, 3
    sizes = np.full(M // 2 + 1, 2, np.int64)
    sizes[-1] = 1
    gene_start = _gene_start(sizes)
    assert gene_start[-1] == M + 1 and M * 4 > STAGE_BYTES
    tm = rng.gamma(0.8, 5.0, (M, n)).astype(F32)
    st, _ = _check(ctx, oracle, tm, _l_bars(rng, n), gene_start, 0)
    assert st.blocks == 1 and st.resident == 1
    assert M // 2 > 65_535 and (M + 31) // 32 > 65_535


def test_push_patterns(ctx, oracle):
    """M = 4 096 (2 048 rows per stage): a push of exactly one stage, one of a stage plus a row, single samples in
    reverse order, a push of no samples, then 8 threads pushing interleaved ranges at once through both stages"""
    rng = np.random.default_rng(4096)
    sizes = rng.integers(1, 8, 1500)
    sizes = sizes[np.cumsum(sizes) <= 4096]
    sizes = np.append(sizes, 4096 - sizes.sum())
    gene_start = _gene_start(sizes[sizes > 0])
    M, n = 4096, 9000
    per = STAGE_BYTES // (4 * M)
    assert per == 2048
    tm = rng.gamma(0.5, 10.0, (M, n)).astype(F32)
    sm = np.ascontiguousarray(tm.T)
    l_bars = _l_bars(rng, n)

    def push(ctx, tm_, lb):
        ctx.ci_push(sm[:per], lb[:per], 0)
        ctx.ci_push(sm[per:2 * per + 1], lb[per:2 * per + 1], per)
        single = range(2 * per + 1, 2 * per + 101)
        for k in reversed(single):
            ctx.ci_push(sm[k:k + 1], lb[k:k + 1], k)
        ctx.ci_push(sm[:0], lb[:0], 2 * per + 101)
        rest = list(range(2 * per + 101, n, 173))
        errors = []

        def worker(t):
            try:
                for a in rest[t::8]:
                    b = min(n, a + 173)
                    ctx.ci_push(sm[a:b], lb[a:b], a)
            except Exception as e:  # noqa: BLE001 - reported below
                errors.append(e)
        threads = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors

    st, _ = _check(ctx, oracle, tm, l_bars, gene_start, cp.threshold(0.95, n), push=push)
    assert st.resident == 1


def _budget_case(rng):
    sizes = np.array([3, 1, 7, 2, 1, 4, 1, 1, 5, 2, 6, 1, 3, 2, 1, 4, 2, 2, 1, 3])
    gene_start = _gene_start(sizes)
    n = 1000
    tm = rng.gamma(0.5, 10.0, (gene_start[-1] - 1, n)).astype(F32)
    tm[5] = 0
    return gene_start, n, tm, _l_bars(rng, n)


def test_budget_edges(ctx, oracle):
    """the budget at the resident threshold and one byte below (same bits either way), a budget whose rows_cap is the
    largest gene's rows (that gene alone fills its block), and one that holds every row (a single block)"""
    rng = np.random.default_rng(7)
    gene_start, n, tm, l_bars = _budget_case(rng)
    M = gene_start[-1] - 1
    thr = cp.threshold(0.95, n)
    max_rows = int(cp.gene_rows(gene_start).max())
    fixed = 20 * n + (1 << 20)
    at = 4 * n * M + fixed + max_rows * 8 * n
    host_exact = fixed + max_rows * 12 * n
    assert host_exact < at - 1
    cases = [(at, True), (at - 1, False), (host_exact, False), (1 << 36, True)]
    for budget, resident in cases:
        st, _ = _check(ctx, oracle, tm, l_bars, gene_start, thr, budget=budget)
        want_res, rows_cap, mr, all_rows = cp.block_rule(gene_start, n, budget)
        assert want_res == resident and st.resident == int(resident)
        blocks = cp.blocks(gene_start, rows_cap)
        assert st.blocks == len(blocks)
        if budget in (at, host_exact):
            assert rows_cap == max_rows and max_rows in blocks
        if budget == 1 << 36:
            assert rows_cap == all_rows and st.blocks == 1


def _allele_case(rng, n):
    """genes of 1 - 6 alleles, isoforms of 1 - 3 alleles inside them"""
    sizes = rng.integers(1, 7, 24)
    gene_start = _gene_start(sizes)
    iso = [1]
    for a, b in zip(gene_start, gene_start[1:]):
        j = a
        while j < b:
            j = min(b, j + int(rng.integers(1, 4)))
            iso.append(j)
    M = gene_start[-1] - 1
    tm = rng.gamma(0.5, 10.0, (M, n)).astype(F32)
    tm[rng.integers(0, M, 4)] = 0
    return gene_start, iso, tm


@pytest.mark.parametrize("threads", [1, 2, 3, 8, 1000])
def test_allele_specific(ctx, oracle, threads):
    """the running isoform sums, sorted in place at each isoform with several alleles and restarted at each Phase II
    range (the host's ranges for -p threads; -p > M leaves empty ranges), one-allele isoforms copying their allele, and
    the chain carried across blocks with the matrix in host memory"""
    rng = np.random.default_rng(threads)
    n = 601
    gene_start, iso, tm = _allele_case(rng, n)
    M = gene_start[-1] - 1
    parts = cp.parts(gene_start, threads)
    widths = np.diff(iso)
    assert (widths == 1).any() and (widths > 1).any()
    if threads > M:
        assert (np.diff(parts) == 0).any()
    l_bars = _l_bars(rng, n)
    thr = cp.threshold(0.95, n)
    st, _ = _check(ctx, oracle, tm, l_bars, gene_start, thr, isoform_start=iso, parts=parts)
    assert st.resident == 1 and st.blocks == 1
    max_rows = int(cp.gene_rows(gene_start).max())
    budget = 20 * n + (1 << 20) + (max_rows + 6) * 12 * n
    st, _ = _check(ctx, oracle, tm, l_bars, gene_start, thr, budget=budget, isoform_start=iso, parts=parts)
    resident, rows_cap, _, _ = cp.block_rule(gene_start, n, budget)
    assert not resident and st.resident == 0 and st.blocks == len(cp.blocks(gene_start, rows_cap)) > 4


@pytest.mark.skipif(not os.path.exists(cp.REF_BIN), reason="oracle/_ref holds no reference tool")
@pytest.mark.parametrize("threads,alleles", [(2, False), (1, True)])
def test_reference_samples(ctx, oracle, tmp_path, threads, alleles):
    """the reference tool's own imd.tmp pushed with arbitrary l_bars: the TPM columns print as the reference printed
    them, and every column equals the restatement's bits"""
    run = cp.reference_run(tmp_path, threads, 50, alleles=alleles)
    rng = np.random.default_rng(threads)
    l_bars = _l_bars(rng, run["n"])
    # the device's outputs equal these bits
    st, (tr, ge, iso) = _check(ctx, oracle, run["samples"], l_bars, run["gene_start"], run["threshold"],
                               isoform_start=run["isoform_start"], parts=run["parts"])
    assert cp.text_rows(tr[:, :3]) == run["rows"]["s.allele_res" if alleles else "s.iso_res"][:3]
    assert cp.text_rows(ge[:, :3]) == run["rows"]["s.gene_res"][:3]
    if alleles:
        assert cp.text_rows(iso[:, :3]) == run["rows"]["s.iso_res"][:3]


def test_refusals(ctx, oracle):
    """push before begin, samples out of range, end twice, a budget below the largest gene (state freed); a begin /
    end cycle afterwards on the same context still matches the restatement"""
    rng = np.random.default_rng(2)
    gene_start, n, tm, l_bars = _budget_case(rng)
    M = gene_start[-1] - 1
    thr = cp.threshold(0.95, n)
    sm = np.ascontiguousarray(tm.T)
    with pytest.raises(RsemB200Error, match="error 2: ci_begin must be called first"):
        ctx.ci_push(sm[:1], l_bars[:1], 0)
    params, keep = _params(gene_start, n, thr)
    ctx.ci_begin(params)
    with pytest.raises(RsemB200Error, match="error 2: samples out of range"):
        ctx.ci_push(sm[:2], l_bars[:2], n - 1)
    ctx.ci_push(sm, l_bars, 0)
    ctx.ci_end(M, len(gene_start) - 1)
    with pytest.raises(RsemB200Error, match="error 2: ci_begin must be called first"):
        ctx.ci_end(M, len(gene_start) - 1)
    max_rows = int(cp.gene_rows(gene_start).max())
    params, keep = _params(gene_start, n, thr, budget=20 * n + (1 << 20) + max_rows * 12 * n - 1)
    with pytest.raises(RsemB200Error, match="error 2: ci_begin: the device budget cannot hold"):
        ctx.ci_begin(params)
    with pytest.raises(RsemB200Error, match="error 2: ci_begin must be called first"):
        ctx.ci_push(sm[:1], l_bars[:1], 0)
    _check(ctx, oracle, tm, l_bars, gene_start, thr)
