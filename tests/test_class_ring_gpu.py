"""The class-layout E-step at the edges of its shared-memory ring and of its batch loop.  Every case goes through the
C ABI, is checked against the CPU oracle and asserts from the layout that it reached the edge it names: tiles per CTA
at the ring's lap boundary, CTAs with a single tile, tiles with several batches per warp next to tiles with fewer
batches than warps, the launch over rows of more than 127 hits, the profiling build with its per-phase cycle
counters, and many launches on one context."""
import numpy as np
import pytest

import synth

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-9, 1e-15
STAGES = 3  # stages of the kernel's shared-memory ring


@pytest.fixture(scope="module")
def ctx(built):
    import rsem_b200
    c = rsem_b200.Context(0)
    c.set_estep_variant(5)
    yield c
    c.close()


@pytest.fixture(scope="module")
def sm_count(built):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _matrix(deg, start, M, seed):
    """rows of deg[i] consecutive transcripts from start[i]: rows with the same (start, deg) form an equivalence class
    (same transcripts, own strands and conprb)"""
    rng = np.random.default_rng(seed)
    deg = np.asarray(deg, np.int64)
    N = len(deg)
    start = np.minimum(np.asarray(start, np.int64), M - deg + 1)
    assert start.min() >= 1
    row_ptr = np.zeros(N + 1, np.uint64)
    row_ptr[1:] = np.cumsum(deg)
    H = int(row_ptr[-1])
    within = np.arange(H) - np.repeat(row_ptr[:-1].astype(np.int64), deg)
    sid = (np.repeat(start, deg) + within).astype(np.int32)
    sid *= np.where(rng.random(H) < 0.5, 1, -1).astype(np.int32)
    conprb = 10.0 ** rng.uniform(-60, -3, size=H)
    tiny = rng.random(H) < 0.02
    conprb[tiny] = 10.0 ** rng.uniform(-320, -295, size=int(tiny.sum()))
    conprb[rng.random(H) < 0.01] = 0.0
    ncpv = 10.0 ** rng.uniform(-80, -40, size=N)
    ncpv[rng.random(N) < 0.05] = 0.0
    return row_ptr, sid, conprb, ncpv


def _classes(N, lo, hi, n_starts, M, seed):
    """N rows of lo..hi hits drawn from n_starts family starts: few, large classes (segments of 8 rows)"""
    rng = np.random.default_rng(seed)
    return rng.integers(lo, hi + 1, N), rng.integers(1, M - hi, n_starts)[rng.integers(0, n_starts, N)]


def _singletons(N, lo, hi, M, seed):
    """N rows of lo..hi hits with starts all over a large M: nearly every row is a class of its own"""
    rng = np.random.default_rng(seed)
    return rng.integers(lo, hi + 1, N), rng.integers(1, M - hi, N)


def _upload(ctx, mat, M):
    row_ptr, sid, conprb, ncpv = mat
    ctx.upload_hits(row_ptr, sid, M)
    ctx.upload_conprb(conprb, ncpv)  # builds the class layout
    info = ctx.class_layout_info()
    assert info["built"] == 1 and info["long_rows"] == 0
    return info


def _run_and_check(ctx, oracle, mat, M, rounds=6):
    """the uploaded matrix: `rounds` EM rounds on the class layout against the oracle; returns theta"""
    row_ptr, sid, conprb, ncpv = mat
    N = len(ncpv)
    n0 = N / 20
    theta0 = synth.init_theta(M, n0, N + n0)
    ctx.set_theta(theta0)
    stats, _ = ctx.em_rounds(1, rounds, rounds + 20, 10000, n0)
    theta = ctx.get_theta()
    theta_ref, stats_ref, _ = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 1, rounds, rounds + 20, 10000)
    big = theta_ref >= 1e-7
    assert np.all(np.abs(theta[big] - theta_ref[big]) <= RTOL * theta_ref[big])
    assert np.all(np.abs(theta[~big] - theta_ref[~big]) <= ATOL + RTOL * theta_ref[~big])
    assert len(stats) == rounds
    for (s, b, t), (s2, b2, t2) in zip(stats, stats_ref):
        assert abs(s - s2) <= 1e-9 * s2
        assert abs(b - b2) <= 1e-6 * b2 + 1e-12
        assert abs(t - t2) <= 2
    return theta


def _sized(ctx, lo, hi, M=3000, seed=11):
    """a matrix of degree-20 classes whose layout has lo..hi tiles: the row count is fitted on the built layout"""
    N = max(200, int((lo + hi) / 2 * 280))  # about 280 such rows per tile
    for _ in range(6):
        mat = _matrix(*_classes(N, 17, 23, 400, M, seed), M, seed)
        info = _upload(ctx, mat, M)
        if lo <= info["tiles"] <= hi:
            return mat, info
        N = max(50, int(N * (lo + hi) / 2 / info["tiles"]))
    pytest.fail(f"no matrix with {lo}..{hi} tiles found (last: {info['tiles']} tiles from {N} rows)")


@pytest.mark.parametrize("per_cta", [1, STAGES, STAGES + 1])
def test_tiles_per_cta_at_the_ring_lap(ctx, oracle, sm_count, per_cta):
    """one tile in all; then every CTA with exactly as many tiles as the ring has stages (each stage used once); then the
    first CTAs with one more (their fourth tile is the first refill: the parity of the barriers flips)"""
    if per_cta == 1:
        mat, info = _sized(ctx, 1, 1)
    else:
        lo = (per_cta - 1) * sm_count + 1
        mat, info = _sized(ctx, lo + sm_count // 8, lo + sm_count - 1 - sm_count // 8)
        assert (info["tiles"] - 1) // sm_count + 1 == per_cta  # tiles of CTA 0: k = 0, sm_count, 2 sm_count, ...
    assert info["tiles_main"] == info["tiles"]
    _run_and_check(ctx, oracle, mat, 3000)
    assert ctx.estep_cta_times().size == min(sm_count, info["tiles"])


def test_fewer_tiles_than_sms(ctx, oracle, sm_count):
    """every CTA has a single tile and some SMs have none"""
    mat, info = _sized(ctx, 8, sm_count // 2)
    _run_and_check(ctx, oracle, mat, 3000)
    assert ctx.estep_cta_times().size == info["tiles"] < sm_count


def test_batches_of_different_configurations(ctx, oracle, sm_count):
    """rows of 1-3 hits in classes of their own (one lane per segment, several batches per warp and tile) and classes
    of ~20-hit rows (8 lanes per segment, fewer batches in a tile than warps, so some warps pass a tile without work)
    in one matrix: where the sorted stream changes degree, a warp's consecutive batches use different lane mappings"""
    M = 400000
    short = _singletons(150000, 1, 3, M, 5)
    wide = _classes(60000, 18, 22, 300, M, 6)
    i_short = _upload(ctx, _matrix(*short, M, 7), M)
    assert i_short["batches"] > 2 * 15 * i_short["tiles"]  # more than two batches per warp in a tile
    i_wide = _upload(ctx, _matrix(*wide, M, 7), M)
    assert i_wide["batches"] < 15 * i_wide["tiles"]  # fewer batches than consumer warps in a tile
    mat = _matrix(np.concatenate([short[0], wide[0]]), np.concatenate([short[1], wide[1]]), M, 7)
    info = _upload(ctx, mat, M)
    assert info["tiles"] > sm_count and info["tiles_main"] == info["tiles"]
    _run_and_check(ctx, oracle, mat, M)


def test_rows_beyond_127_hits_next_to_short_rows(ctx, oracle, sm_count):
    """rows of 128-400 hits run in the launch of their own, over CTAs with several tiles; its extra columns read ids
    from the stage during the row walk"""
    M = 6000
    longr = _classes(9000, 128, 400, 120, M, 1)
    short = _classes(40000, 1, 30, 2000, M, 2)
    mat = _matrix(np.concatenate([short[0], longr[0]]), np.concatenate([short[1], longr[1]]), M, 3)
    info = _upload(ctx, mat, M)
    assert info["tiles_main"] > 0 and info["tiles"] - info["tiles_main"] > 2 * sm_count  # CTAs with >= 3 tail tiles
    _run_and_check(ctx, oracle, mat, M)


def test_profiling_counts_the_phases(ctx, oracle, sm_count):
    mat, info = _sized(ctx, 3 * sm_count, 5 * sm_count)
    theta = _run_and_check(ctx, oracle, mat, 3000)
    assert ctx.estep_wait_times().size == 0  # the latest launch ran without profiling
    ctx.set_profiling(True)
    try:
        _upload(ctx, mat, 3000)
        theta_prof = _run_and_check(ctx, oracle, mat, 3000)
        w = ctx.estep_wait_times().astype(np.float64)
    finally:
        ctx.set_profiling(False)
    big = theta >= 1e-7
    assert np.all(np.abs(theta_prof[big] - theta[big]) <= 1e-12 * theta[big])
    assert w.shape == (sm_count, 8)
    warps, phases, busy_cycles = w[:, 2], w[:, 3:7], w[:, 7]
    assert np.all(warps == warps[0]) and warps[0] >= 1
    assert np.all(phases > 0)  # front, rows, flush, hand-over: summed over the CTA's consumer warps
    assert np.all(phases.sum(axis=1) <= warps * busy_cycles)


def test_thirty_rounds_and_the_stop_flag(ctx, oracle, sm_count):
    """the ring and its barriers are set up again by every launch; once the device has decided to stop, the launches
    already queued return at once and the result is that of the oracle's last round"""
    mat, info = _sized(ctx, 3 * sm_count + 1, 4 * sm_count)
    _run_and_check(ctx, oracle, mat, 3000, rounds=30)
    row_ptr, sid, conprb, ncpv = synth.random_matrix(3000, 40, 2, seed=5, tiny_frac=0, family=False)
    n0 = 100.0
    theta0 = synth.init_theta(40, n0, 3100)
    _upload(ctx, (row_ptr, sid, conprb, ncpv), 40)
    ctx.set_theta(theta0)
    stats, stopped = ctx.em_rounds(1, 400, 5, 300, n0)
    theta_ref, stats_ref, stopped_ref = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 1, 400, 5, 300)
    assert stopped and stopped_ref and len(stats) == len(stats_ref) < 300
    theta = ctx.get_theta()
    big = theta_ref >= 1e-7
    assert np.all(np.abs(theta[big] - theta_ref[big]) <= RTOL * theta_ref[big])
