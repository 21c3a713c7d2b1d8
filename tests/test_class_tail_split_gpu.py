"""The class-layout E-step runs rows of more than 127 hits (more columns than a 32-lane group holds in registers) in a
launch of their own, over tiles that hold nothing else; rows of more than 2047 hits keep their CSR launch.  Every
split is checked against the CPU oracle: rows right at the 127 / 128 and 2047 / 2048 boundaries, a matrix with only
the second launch, and one with only the first."""
import numpy as np
import pytest

import synth

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-9, 1e-15


@pytest.fixture(scope="module")
def ctx(built):
    import rsem_b200
    c = rsem_b200.Context(0)
    yield c
    c.close()


def _matrix(degrees, M, seed):
    """degrees: [(hits per read, distinct transcript lists, reads per list)]; reads of one list share its transcripts
    (an equivalence class) but not their strands or conprb; rows shuffled"""
    rng = np.random.default_rng(seed)
    lists = []
    for d, n_lists, dup in degrees:
        for _ in range(n_lists):
            ids = rng.choice(np.arange(1, M + 1), size=d, replace=False).astype(np.int32)
            lists += [ids] * dup
    order = rng.permutation(len(lists))
    rows = [lists[i] * np.where(rng.random(len(lists[i])) < 0.5, 1, -1).astype(np.int32) for i in order]
    degs = np.array([len(r) for r in rows], np.uint64)
    row_ptr = np.zeros(len(rows) + 1, np.uint64)
    row_ptr[1:] = np.cumsum(degs)
    sid = np.concatenate(rows).astype(np.int32)
    H, N = len(sid), len(rows)
    conprb = 10.0 ** rng.uniform(-60, -3, size=H)
    conprb[rng.random(H) < 0.02] = 10.0 ** rng.uniform(-320, -295, size=1)
    conprb[rng.random(H) < 0.01] = 0.0
    ncpv = 10.0 ** rng.uniform(-80, -40, size=N)
    ncpv[rng.random(N) < 0.05] = 0.0
    return row_ptr, sid, conprb, ncpv


def _short(rng_seed, n_lists):
    rng = np.random.default_rng(rng_seed)
    return [(int(d), 1, int(k)) for d, k in zip(1 + rng.poisson(9, n_lists), rng.integers(1, 25, n_lists))]


CASES = {
    # rows at both boundaries between short rows: both class-layout launches and the long-row launch run
    "mixed": (_short(1, 2000) + [(d, 3, 11) for d in (126, 127, 128, 129, 200)] + [(d, 1, 1) for d in (126, 127, 128, 129)]
              + [(2047, 2, 3), (2047, 1, 1), (2048, 1, 2)]),
    # every row has at least 128 hits: the first launch has no tiles
    "tail_only": [(d, 4, 9) for d in (128, 129, 150, 200, 300, 700)] + [(d, 2, 1) for d in (128, 255, 256, 1000)],
    # every row has at most 127 hits: no second launch
    "main_only": _short(2, 2000) + [(d, 3, 11) for d in (64, 100, 126, 127)] + [(127, 2, 1)],
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_tail_split_matches_oracle(ctx, oracle, name):
    M = 5000
    row_ptr, sid, conprb, ncpv = _matrix(CASES[name], M, seed=len(name))
    N = len(ncpv)
    n0 = N / 20
    theta0 = synth.init_theta(M, n0, N + n0)
    ctx.set_estep_variant(5)
    ctx.upload_hits(row_ptr, sid, M)
    ctx.upload_conprb(conprb, ncpv)
    ctx.set_theta(theta0)
    stats, _ = ctx.em_rounds(1, 6, 20, 10000, n0)
    info = ctx.class_layout_info()
    busy = ctx.estep_cta_times()
    theta = ctx.get_theta()
    ctx.set_estep_variant(0)
    degs = np.diff(row_ptr.astype(np.int64))
    n_long = int((degs > 2047).sum())
    assert info["built"] == 1 and info["long_rows"] == n_long and info["rows"] == N - n_long
    if name == "mixed":
        assert n_long == 2 and 0 < info["tiles_main"] < info["tiles"]
    elif name == "tail_only":
        assert n_long == 0 and info["tiles_main"] == 0 < info["tiles"]
    else:
        assert n_long == 0 and info["tiles_main"] == info["tiles"] > 0
    # per-CTA busy times come from the launch over the main tiles only
    assert (busy.size > 0) == (info["tiles_main"] > 0)
    theta_ref, stats_ref, _ = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 1, 6, 20, 10000)
    big = theta_ref >= 1e-7
    assert np.all(np.abs(theta[big] - theta_ref[big]) <= RTOL * theta_ref[big])
    assert np.all(np.abs(theta[~big] - theta_ref[~big]) <= ATOL + RTOL * theta_ref[~big])
    assert len(stats) == 6
    for (s, b, t), (s2, b2, t2) in zip(stats, stats_ref):
        assert abs(s - s2) <= 1e-9 * s2
        assert abs(b - b2) <= 1e-6 * b2 + 1e-12
        assert abs(t - t2) <= 2
