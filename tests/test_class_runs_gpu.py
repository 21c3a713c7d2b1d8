"""The class layout stores the ids of a batch whose rows hit consecutive transcripts ("runs": first, first + 1, ...,
first + d - 1) as one first per segment, or one per batch when its segments belong to one class, and the E-step forms
the ids from them.  Rows that are not runs keep every id.  Every case is checked against the CPU oracle, together with
the round the EM stops at: runs at the column counts where the lane-group configuration changes, rows that are not
runs (permuted, descending, a transcript hit twice, a gap) next to runs of the same shape, mostly singleton classes,
and rows of more than 127 hits, which keep their ids and their own launch.  The layout accounting is checked on
matrices whose batches are known in advance."""
import numpy as np
import pytest

import synth

pytestmark = pytest.mark.gpu

RTOL = 1e-9
# d + 1 = 3, 4, 5, 8, 9, 16, 17, 32, 33, 64, 65, 128: the column counts at which lanes per segment or slots per lane change
SWITCH_DEGREES = (2, 3, 4, 7, 8, 15, 16, 31, 32, 63, 64, 127)


@pytest.fixture(scope="module")
def ctx(built):
    import rsem_b200
    c = rsem_b200.Context(0)
    c.set_estep_variant(5)
    yield c
    c.close()


def _lanes(d):
    w = d + 1
    return 1 if w <= 4 else 2 if w <= 8 else 4 if w <= 16 else 8 if w <= 32 else 16 if w <= 64 else 32


def _matrix(lists, seed):
    """lists: [(transcript ids, reads)]; the reads of one list form a class (random strands and conprb); rows shuffled"""
    rng = np.random.default_rng(seed)
    rows = [np.asarray(ids, np.int32) for ids, n in lists for _ in range(n)]
    order = rng.permutation(len(rows))
    rows = [rows[i] * np.where(rng.random(len(rows[i])) < 0.5, 1, -1).astype(np.int32) for i in order]
    row_ptr = np.zeros(len(rows) + 1, np.uint64)
    row_ptr[1:] = np.cumsum([len(r) for r in rows])
    sid = np.concatenate(rows).astype(np.int32)
    H, N = len(sid), len(rows)
    conprb = 10.0 ** rng.uniform(-60, -3, size=H)
    conprb[rng.random(H) < 0.02] = 10.0 ** rng.uniform(-320, -295, size=1)
    conprb[rng.random(H) < 0.01] = 0.0
    ncpv = 10.0 ** rng.uniform(-80, -40, size=N)
    ncpv[rng.random(N) < 0.05] = 0.0
    return row_ptr, sid, conprb, ncpv


def _run(first, d):
    return np.arange(first, first + d)


def _runs_at_switch_degrees(M, rng):
    lists = []
    for d in SWITCH_DEGREES:
        P = 32 // _lanes(d)
        starts = rng.integers(1, M - d + 2, size=40)
        lists += [(_run(s, d), 1) for s in starts[:20]]          # single-row segments
        lists += [(_run(s, d), 8) for s in starts[20:30]]        # one full segment per class
        lists += [(_run(s, d), 8 * P * 2 + 3) for s in starts[30:32]]  # one-class batches, and a 3-row segment
        lists += [(_run(s, d), int(k)) for s, k in zip(starts[32:], rng.integers(2, 20, size=8))]
        lists += [(_run(M - d + 1, d), 5), (_run(1, d), 2)]  # runs that end at transcript M and start at 1
    return lists


def _not_runs(M, rng):
    lists = []
    for d in SWITCH_DEGREES:
        for _ in range(6):
            ids = _run(int(rng.integers(2, M - d - 1)), d)
            permuted = rng.permutation(ids)
            while np.all(np.diff(permuted) == 1):
                permuted = rng.permutation(ids)
            lists.append((permuted, int(rng.integers(1, 12))))
            lists.append((ids[::-1].copy(), int(rng.integers(1, 12))))  # descending
            twice = ids.copy()
            twice[-1] = twice[-2]  # the last transcript hit twice
            lists.append((twice, int(rng.integers(1, 12))))
            gap = ids.copy()
            gap[-1] += 1  # consecutive but for one gap
            lists.append((gap, int(rng.integers(1, 12))))
    return lists


def _singletons(M, rng):
    """mostly one read per transcript list, degrees 1..40"""
    lists = [(_run(int(s), int(d)), 1)
             for d, s in zip(rng.integers(1, 41, 20000), rng.integers(1, M - 40, 20000))]
    return lists + [(_run(int(s), 12), 9) for s in rng.integers(1, M - 12, 200)]


def _with_tail(M, rng):
    lists = [(_run(int(s), int(d)), int(k))
             for d, s, k in zip(1 + rng.poisson(15, 3000), rng.integers(1, M - 200, 3000), rng.integers(1, 20, 3000))]
    lists += [(_run(int(s), int(d)), int(k))
              for d, s, k in zip(rng.integers(128, 300, 300), rng.integers(1, M - 300, 300), rng.integers(1, 6, 300))]
    return lists


CASES = {
    "runs": _runs_at_switch_degrees,
    "not_runs": _not_runs,
    "runs_and_not_runs": lambda M, rng: _runs_at_switch_degrees(M, rng) + _not_runs(M, rng),
    "singletons": _singletons,
    "runs_and_tail": _with_tail,
}


def _check(ctx, oracle, mat, M, rounds):
    row_ptr, sid, conprb, ncpv = mat
    N = len(ncpv)
    n0 = N / 20
    theta0 = synth.init_theta(M, n0, N + n0)
    ctx.set_theta(theta0)
    # rounds >= 12 run on the class layout; min_round 13 lets the EM stop as soon as it has converged
    stats, stopped = ctx.em_rounds(12, rounds, 13, 10000, n0)
    theta_ref, stats_ref, stopped_ref = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 12, rounds, 13, 10000)
    assert stopped == stopped_ref and len(stats) == len(stats_ref)
    theta = ctx.get_theta()
    big = theta_ref >= 1e-7
    assert np.all(np.abs(theta[big] - theta_ref[big]) <= RTOL * theta_ref[big])


def _is_run(ids):
    a = np.abs(ids.astype(np.int64))
    return len(a) >= 1 and np.all(np.diff(a) == 1)


@pytest.mark.parametrize("name", sorted(CASES))
def test_runs_match_oracle(ctx, oracle, name):
    M = 4000
    rng = np.random.default_rng(len(name))
    mat = _matrix(CASES[name](M, rng), seed=len(name) + 1)
    row_ptr, sid = mat[0], mat[1]
    ctx.upload_hits(row_ptr, sid, M)
    ctx.upload_conprb(mat[2], mat[3])
    info = ctx.class_layout_info()
    assert info["built"] == 1
    rp = row_ptr.astype(np.int64)
    degs = np.diff(rp)
    run_hits = sum(int(degs[i]) for i in range(len(degs)) if degs[i] <= 127 and _is_run(sid[rp[i]:rp[i + 1]]))
    assert info["run_hits"] == run_hits
    if name == "runs":
        assert run_hits == int(row_ptr[-1])
    if name == "not_runs":
        assert run_hits == 0
    if name == "runs_and_tail":
        assert 0 < info["tiles_main"] < info["tiles"]
    _check(ctx, oracle, mat, M, 60)


def test_layout_stores_one_first_per_segment_or_batch(ctx):
    """degrees whose classes all have 16 P rows (two full segments per batch, every batch of one class): one first per
    batch; degrees of singleton classes: one first per segment; the same rows permuted: every id"""
    M = 6000
    rng = np.random.default_rng(7)
    one_class, single = (3, 9, 40, 127), (5, 20, 63, 100)
    lists = []
    batches = segments = firsts = 0
    for d in one_class:
        P = 32 // _lanes(d)
        for s in rng.choice(np.arange(1, M - d + 2), size=3, replace=False):
            lists.append((_run(int(s), d), 16 * P))
        segments += 3 * 2 * P
        batches += 3 * 2
        firsts += 3 * 2
    for d in single:
        P = 32 // _lanes(d)
        n = 100
        lists += [(_run(int(s), d), 1) for s in rng.choice(np.arange(1, M - d + 2), size=n, replace=False)]
        segments += n
        batches += -(-n // P)
        firsts += n
    row_ptr, sid, conprb, ncpv = _matrix(lists, seed=8)
    ctx.upload_hits(row_ptr, sid, M)
    ctx.upload_conprb(conprb, ncpv)
    info = ctx.class_layout_info()
    H = int(row_ptr[-1])
    assert (info["segments"], info["batches"], info["ids"], info["run_hits"]) == (segments, batches, firsts, H)
    assert info["bytes_per_round"] == 8 * info["vals"] + 4 * firsts + 16 * batches

    permuted = [(ids[::-1].copy(), n) for ids, n in lists]  # descending: no run, every id stored
    row_ptr, sid, conprb, ncpv = _matrix(permuted, seed=8)
    ctx.upload_hits(row_ptr, sid, M)
    ctx.upload_conprb(conprb, ncpv)
    info = ctx.class_layout_info()
    # one-class batches keep one id list per batch, other batches one per segment
    assert info["run_hits"] == 0 and info["ids"] == sum(3 * 2 * d for d in one_class) + sum(100 * d for d in single)
