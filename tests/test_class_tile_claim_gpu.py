"""The class-layout E-step's CTAs claim tiles from a counter in global memory that the last CTA of a launch sets back
to zero.  These cases check that the counter is right for the next launch in the situations that end a launch in
different ways: the main launch followed by the launch over rows of more than 127 hits on the same counter, launches
that return at once because the device has decided to stop, and a new layout built on the same context afterwards."""
import numpy as np
import pytest

import synth

pytestmark = pytest.mark.gpu

RTOL = 1e-9


@pytest.fixture(scope="module")
def ctx(built):
    import rsem_b200
    c = rsem_b200.Context(0)
    c.set_estep_variant(5)
    yield c
    c.close()


def _matrix(deg, start, M, seed):
    """rows of deg[i] consecutive transcripts from start[i]"""
    rng = np.random.default_rng(seed)
    deg = np.asarray(deg, np.int64)
    row_ptr = np.zeros(len(deg) + 1, np.uint64)
    row_ptr[1:] = np.cumsum(deg)
    H = int(row_ptr[-1])
    within = np.arange(H) - np.repeat(row_ptr[:-1].astype(np.int64), deg)
    sid = (np.repeat(np.asarray(start, np.int64), deg) + within).astype(np.int32)
    sid *= np.where(rng.random(H) < 0.5, 1, -1).astype(np.int32)
    conprb = 10.0 ** rng.uniform(-60, -3, size=H)
    ncpv = 10.0 ** rng.uniform(-80, -40, size=len(deg))
    return row_ptr, sid, conprb, ncpv


def _short_and_long(M, seed):
    rng = np.random.default_rng(seed)
    deg = np.r_[rng.integers(1, 40, 60000), rng.integers(128, 300, 6000)]
    start = rng.integers(1, M - 300, len(deg))
    return _matrix(deg, start, M, seed)


def _check(ctx, oracle, mat, M, first, rounds, min_round, max_round, n0):
    row_ptr, sid, conprb, ncpv = mat
    theta0 = synth.init_theta(M, n0, len(ncpv) + n0)
    ctx.set_theta(theta0)
    stats, stopped = ctx.em_rounds(first, rounds, min_round, max_round, n0)
    theta_ref, stats_ref, stopped_ref = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, first, rounds,
                                                         min_round, max_round)
    assert stopped == stopped_ref and len(stats) == len(stats_ref)
    theta = ctx.get_theta()
    big = theta_ref >= 1e-7
    assert np.all(np.abs(theta[big] - theta_ref[big]) <= RTOL * theta_ref[big])
    return stopped, len(stats)


def test_main_and_tail_launches_share_the_counter(ctx, oracle):
    M = 5000
    mat = _short_and_long(M, 1)
    ctx.upload_hits(mat[0], mat[1], M)
    ctx.upload_conprb(mat[2], mat[3])
    info = ctx.class_layout_info()
    assert info["built"] == 1 and 0 < info["tiles_main"] < info["tiles"]
    # rounds >= 12 run on the class layout: every round is a main launch, then a tail launch
    _check(ctx, oracle, mat, M, 12, 20, 10000, 10000, len(mat[3]) / 20)


def test_launches_after_the_stop_and_a_new_layout(ctx, oracle):
    """once the device has decided to stop, the launches still queued return without claiming; the next em_rounds on
    the same layout, and then on a new layout, start from tile 0"""
    row_ptr, sid, conprb, ncpv = synth.random_matrix(3000, 40, 2, seed=5, tiny_frac=0, family=False)
    mat = (row_ptr, sid, conprb, ncpv)
    ctx.upload_hits(row_ptr, sid, 40)
    ctx.upload_conprb(conprb, ncpv)
    assert ctx.class_layout_info()["tiles"] >= 1
    stopped, n = _check(ctx, oracle, mat, 40, 1, 400, 5, 300, 100.0)
    assert stopped and n < 300
    _check(ctx, oracle, mat, 40, 12, 8, 10000, 10000, 100.0)
    M = 5000
    mat = _short_and_long(M, 2)
    ctx.upload_hits(mat[0], mat[1], M)
    ctx.upload_conprb(mat[2], mat[3])
    _check(ctx, oracle, mat, M, 12, 6, 10000, 10000, len(mat[3]) / 20)
