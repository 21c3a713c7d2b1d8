"""The class layout's segment rule: a class of n rows and degree d is cut into segments of seg_rows(d, n) rows
(class_kernels.cu).  Classes of at least 8 P rows (P = 32 / G segments per batch) keep the 8-row cut and fill one-class
batches; smaller classes are cut into ceil(n / cap) segments, cap = max(rows_cap(d, 8), min(8 P - 1, V / (P (d + 1))))
with the batch value budget V, so that a class pays as few theta gathers and reductions as a batch allows.

The CPU half restates the rule and the layout built on it (row keys, classes, segments, batches, ids) in numpy and
checks the rule's edges for every lane-group configuration and for the rows of more than 127 hits.  The GPU half
uploads matrices at those edges, asserts that class_layout_info() equals the restatement, and checks the EM rounds
against the CPU oracle; one matrix with power-of-two theta, conprb and row sums checks a class-layout round bit for
bit."""
import numpy as np
import pytest

import synth

gpu = pytest.mark.gpu

RTOL, ATOL = 1e-9, 1e-15

# class_kernels.cu constants
K_LONG_DEG = 2047
MAX_BATCH_VALS = 4096
BUDGET = 2048  # kBatchValBudget
STAGE_BYTES = 64 * 1024
TAIL_CFG = 12

# one degree per configuration 0..11 (G = 1, 2, 4, 8, 16, 32 lanes per segment; 3 or 4 slots per lane), then the tail
CFG_DEGREES = (1, 3, 4, 7, 8, 15, 19, 31, 32, 63, 64, 127, 200)


def lanes(d):
    w = d + 1
    return 1 if w <= 4 else 2 if w <= 8 else 4 if w <= 16 else 8 if w <= 32 else 16 if w <= 64 else 32


def cfg_of(d):
    if d + 1 > 128:
        return TAIL_CFG
    G = lanes(d)
    return 2 * (G.bit_length() - 1) + (1 if d + 1 > 3 * G else 0)


def rows_cap(d, R):
    P = 32 // lanes(d)
    return max(1, min(MAX_BATCH_VALS // (P * (d + 1)), R))


def cap_small(d):
    """rows per segment of a class smaller than 8 P"""
    P = 32 // lanes(d)
    return max(rows_cap(d, 8), min(8 * P - 1, BUDGET // (P * (d + 1))))


def seg_rows(d, n):
    P = 32 // lanes(d)
    return rows_cap(d, 8) if n >= 8 * P else cap_small(d)


# ------------------------------------------------------------------------------------------------------------------
# restatement of class_build
# ------------------------------------------------------------------------------------------------------------------
M64 = (1 << 64) - 1


def _mix(i, c):
    x = (i * 0x9E3779B97F4A7C15 + (c + 1) * 0xC2B2AE3D27D4EB4F) & M64
    x ^= x >> 29
    x = (x * 0xBF58476D1CE4E5B9) & M64
    return x ^ (x >> 32)


def restate(row_ptr, sid, R=0):
    """class_layout_info() of the matrix: R = 0 the default cut (seg_rows), R > 0 segments of rows_cap(d, R) rows"""
    rp = np.asarray(row_ptr).astype(np.int64)
    a = np.abs(np.asarray(sid).astype(np.int64))
    N = len(rp) - 1
    lists, keys = [], []
    for i in range(N):
        ids = a[rp[i]:rp[i + 1]]
        d = len(ids)
        lists.append(tuple(int(x) for x in ids))
        if d > K_LONG_DEG:
            keys.append(1 << 59)
        else:
            h = sum(_mix(int(x), c) for c, x in enumerate(ids)) & M64
            keys.append((d << 48) | (h >> 16))
    order = sorted(range(N), key=lambda i: keys[i])  # stable, as the radix sort
    order = [i for i in order if keys[i] != 1 << 59]
    segs = []  # (key2, class index, degree, rows)
    p = 0
    while p < len(order):
        q = p + 1
        while q < len(order) and keys[order[q]] == keys[order[p]] and lists[order[q]] == lists[order[p]]:
            q += 1
        ids = lists[order[p]]
        d, n = len(ids), q - p
        r = rows_cap(d, R) if R else seg_rows(d, n)
        run = d >= 1 and cfg_of(d) != TAIL_CFG and all(ids[c] == ids[0] + c for c in range(d))
        for s in range(0, n, r):
            rows = min(r, n - s)
            segs.append(((d << 9) | (256 if run else 0) | (255 - rows), p, d, rows, run))
        p = q
    segs.sort(key=lambda s: s[0])  # stable
    batches = ids_n = vals = run_hits = max_bytes = 0
    f = 0
    while f < len(segs):
        g = f
        while g < len(segs) and segs[g][0] == segs[f][0]:
            g += 1
        d, rows, run = segs[f][2], segs[f][3], segs[f][4]
        P = 32 // lanes(d)
        for b in range(f, g, P):
            chunk = segs[b:min(b + P, g)]
            nsb = len(chunk)
            same = all(s[1] == chunk[0][1] for s in chunk)
            per_seg = 1 if run else d
            batches += 1
            ids_n += per_seg if same else nsb * per_seg
            nv = nsb * rows * (d + 1)
            vals += nv
            max_bytes = max(max_bytes, 8 * nv + 4 * nsb * per_seg + 16)
            if run:
                run_hits += nsb * rows * d
        f = g
    return dict(rows=len(order), long_rows=N - len(order), segments=len(segs), batches=batches, vals=vals, ids=ids_n,
                run_hits=run_hits, bytes_per_round=8 * vals + 4 * ids_n + 16 * batches, max_batch_bytes=max_bytes)


def edge_sizes(d):
    """class sizes at the rule's edges for degree d"""
    P = 32 // lanes(d)
    c = cap_small(d)
    return sorted({1, 2, 8 * P - 1, 8 * P, c, c + 1, 8 * P + 3, 3 * 8 * P + c})


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
    conprb[rng.random(H) < 0.01] = 0.0
    ncpv = 10.0 ** rng.uniform(-80, -40, size=N)
    ncpv[rng.random(N) < 0.05] = 0.0
    return row_ptr, sid, conprb, ncpv


def edge_lists(d, M, rng):
    """for every edge size: two run classes and one class whose ids are not a run (descending)"""
    lists = []
    for n in edge_sizes(d):
        for k in range(3):
            s = int(rng.integers(1, M - d + 1))
            ids = np.arange(s, s + d)
            lists.append((ids[::-1].copy() if k == 2 and d > 1 else ids, n))
    return lists


# ------------------------------------------------------------------------------------------------------------------
# CPU half
# ------------------------------------------------------------------------------------------------------------------
def test_rule_edges_in_every_configuration():
    assert [cfg_of(d) for d in CFG_DEGREES] == list(range(13))
    by_batch, by_budget = [], []
    for d in CFG_DEGREES:
        P = 32 // lanes(d)
        c = cap_small(d)
        cuts = {n: -(-n // seg_rows(d, n)) for n in edge_sizes(d)}
        assert cuts[8 * P] == P                          # 8-row cut: one full one-class batch
        assert cuts[c] == 1
        if P == 1:
            assert c == rows_cap(d, 8)
            continue
        assert cuts[c + 1] == 2
        assert seg_rows(d, 8 * P - 1) == c
        if c == 8 * P - 1:
            by_batch.append(d)
            assert cuts[8 * P - 1] == 1
        else:
            by_budget.append(d)
            assert c == BUDGET // (P * (d + 1)) > rows_cap(d, 8)
    assert by_batch == [32, 63]  # 16 lanes per segment: two segments in a batch
    assert by_budget == [1, 3, 4, 7, 8, 15, 19, 31]


def test_rule_never_cuts_more_and_p1_is_unchanged():
    for d in range(1, K_LONG_DEG + 1):
        P = 32 // lanes(d)
        r8 = rows_cap(d, 8)
        for n in range(1, 8 * P + 2):
            r = seg_rows(d, n)
            assert r <= 255 and -(-n // r) <= -(-n // r8)
            assert P * r * (d + 1) <= max(BUDGET, P * r8 * (d + 1)) <= MAX_BATCH_VALS
            if P == 1:  # G = 32 and the rows of more than 127 hits: the 8-row cut
                assert r == r8


@pytest.mark.parametrize("d", CFG_DEGREES)
def test_restatement_of_single_classes(d):
    """one run class per matrix: ceil(n / rows) segments, one batch per P full segments plus the remainder's, one id
    per batch (a one-class batch of runs stores a single first)"""
    P = 32 // lanes(d)
    for n in edge_sizes(d):
        row_ptr, sid, _, _ = _matrix([(np.arange(5, 5 + d), n)], seed=n)
        r = seg_rows(d, n)
        full, rem = divmod(n, r)
        batches = -(-full // P) + (1 if rem else 0)
        run = cfg_of(d) != TAIL_CFG
        ids = batches if run else batches * d
        vals = n * (d + 1)
        got = restate(row_ptr, sid)
        assert (got["segments"], got["batches"], got["ids"], got["vals"]) == (full + (1 if rem else 0), batches, ids, vals)
        assert got["bytes_per_round"] == 8 * vals + 4 * ids + 16 * batches
        assert got["run_hits"] == (n * d if run else 0)
        assert got["max_batch_bytes"] + 256 <= STAGE_BYTES


def test_rule_reduces_segments_of_small_classes():
    """a C3-shaped degree (19, P = 4) with classes of 1..40 rows: fewer segments and batches than the 8-row cut"""
    rng = np.random.default_rng(3)
    lists = [(np.arange(s, s + 19), int(n)) for s, n in zip(rng.integers(1, 5000, 300), rng.integers(1, 41, 300))]
    row_ptr, sid, _, _ = _matrix(lists, seed=4)
    new, old = restate(row_ptr, sid), restate(row_ptr, sid, R=8)
    assert new["vals"] == old["vals"]
    assert new["segments"] < 0.75 * old["segments"] and new["batches"] < old["batches"]


# ------------------------------------------------------------------------------------------------------------------
# GPU half
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx(built):
    import rsem_b200
    c = rsem_b200.Context(0)
    c.set_estep_variant(5)
    yield c
    c.close()


def _upload(ctx, mat, M):
    ctx.upload_hits(mat[0], mat[1], M)
    ctx.upload_conprb(mat[2], mat[3])
    info = ctx.class_layout_info()
    assert info["built"] == 1
    return info


def _assert_info(info, want):
    got = {k: info[k] for k in ("rows", "long_rows", "segments", "batches", "vals", "ids", "run_hits", "bytes_per_round")}
    assert got == {k: want[k] for k in got}


def _check_rounds(ctx, oracle, mat, M, rounds=8):
    row_ptr, sid, conprb, ncpv = mat
    N = len(ncpv)
    n0 = N / 20
    theta0 = synth.init_theta(M, n0, N + n0)
    ctx.set_theta(theta0)
    # rounds >= 12 run on the class layout; min_round 13 lets the EM stop as soon as it has converged
    stats, stopped = ctx.em_rounds(12, rounds, 13, 10000, n0)
    theta_ref, stats_ref, stopped_ref = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 12, rounds, 13, 10000)
    assert stopped == stopped_ref and len(stats) == len(stats_ref)
    for (s, b, t), (s2, b2, t2) in zip(stats, stats_ref):
        assert abs(s - s2) <= 1e-9 * s2
        assert abs(b - b2) <= 1e-6 * b2 + 1e-12
        assert abs(t - t2) <= 2
    theta = ctx.get_theta()
    big = theta_ref >= 1e-7
    assert np.all(np.abs(theta[big] - theta_ref[big]) <= RTOL * theta_ref[big])
    assert np.all(np.abs(theta[~big] - theta_ref[~big]) <= ATOL + RTOL * theta_ref[~big])


@gpu
@pytest.mark.parametrize("d", CFG_DEGREES)
def test_edges_match_restatement_and_oracle(ctx, oracle, monkeypatch, d):
    monkeypatch.delenv("RSEM_B200_CLASS_ROWS", raising=False)
    M = 3000
    mat = _matrix(edge_lists(d, M, np.random.default_rng(d)), seed=d + 1)
    info = _upload(ctx, mat, M)
    _assert_info(info, restate(mat[0], mat[1]))
    _check_rounds(ctx, oracle, mat, M)


@gpu
def test_all_configurations_and_the_fixed_cut(ctx, oracle, monkeypatch):
    """every configuration's edges in one matrix under the default rule; RSEM_B200_CLASS_ROWS=8 selects the 8-row cut"""
    M = 3000
    rng = np.random.default_rng(99)
    lists = [x for d in CFG_DEGREES for x in edge_lists(d, M, rng)]
    mat = _matrix(lists, seed=100)
    monkeypatch.delenv("RSEM_B200_CLASS_ROWS", raising=False)
    info = _upload(ctx, mat, M)
    _assert_info(info, restate(mat[0], mat[1]))
    assert 0 < info["tiles_main"] < info["tiles"]
    _check_rounds(ctx, oracle, mat, M)
    monkeypatch.setenv("RSEM_B200_CLASS_ROWS", "8")
    fixed = _upload(ctx, mat, M)
    _assert_info(fixed, restate(mat[0], mat[1], R=8))
    assert fixed["segments"] > info["segments"]
    _check_rounds(ctx, oracle, mat, M)


def _exact_matrix(lists, seed):
    """the classes of `lists` with powers of two for theta and conprb, and a noise term that tops every row up to a
    power-of-two sum: every weight is dyadic and exact, every count is exact in any summation order"""
    rng = np.random.default_rng(seed)
    M = max(int(np.max(ids)) for ids, _ in lists)
    e = rng.integers(2, 15, M + 1)
    e[0] = 3
    theta = 2.0 ** -e.astype(np.float64)
    rows = [np.asarray(ids, np.int64) for ids, n in lists for _ in range(n)]
    rows = [rows[i] for i in rng.permutation(len(rows))]
    degs = np.array([len(r) for r in rows])
    row_ptr = np.zeros(len(rows) + 1, np.uint64)
    row_ptr[1:] = np.cumsum(degs)
    t = np.concatenate(rows)
    u = rng.integers(0, 17, len(t))                      # products 2^-(10 + u)
    conprb = 2.0 ** (e[t] - 10 - u).astype(np.float64)
    ints = np.left_shift(np.int64(1), 16 - u)          # in units of 2^-26
    rs = np.add.reduceat(ints, row_ptr[:-1].astype(np.int64))
    top = np.left_shift(np.int64(1), np.frexp(rs.astype(np.float64))[1].astype(np.int64))
    ncpv = (top - rs).astype(np.float64) * 2.0 ** -26 * 2.0 ** 3
    sid = (t * np.where(rng.random(len(t)) < 0.5, 1, -1)).astype(np.int32)
    return (row_ptr, sid, conprb, ncpv), theta, M


@gpu
def test_class_round_is_exact(ctx, oracle, monkeypatch):
    """one frozen round on the class layout under the default cut: theta and the round statistics bit for bit"""
    monkeypatch.delenv("RSEM_B200_CLASS_ROWS", raising=False)
    rng = np.random.default_rng(5)
    lists = []
    for d in CFG_DEGREES:
        for n in edge_sizes(d):
            s = int(rng.integers(1, 2000))
            lists.append((np.arange(s, s + d), n))
    mat, theta, M = _exact_matrix(lists, seed=6)
    info = _upload(ctx, mat, M)
    _assert_info(info, restate(mat[0], mat[1]))
    n0 = len(mat[3]) // 16 + 1.0
    c_ref = oracle.estep(*mat, theta)
    th_ref, st_ref = oracle.mstep(c_ref, theta, n0)
    ctx.set_theta(theta)
    stats, stopped = ctx.em_rounds(12, 1, 20, 10000, n0)
    assert not stopped and len(stats) == 1
    assert stats[0] == st_ref
    th = ctx.get_theta()
    bad = np.flatnonzero(th != th_ref)
    assert bad.size == 0, f"{bad.size} differ, first at {bad[:5]}"
