"""K2 (E-step + count accumulation) and K4 (theta update / convergence) against the CPU oracle.

Tolerance: the path is fp64 with an unordered (atomic) accumulation, the reference itself is only
reproducible to ~1e-13 across thread counts (-ffast-math); north_star asks for 1e-6 relative on
theta.  We assert 1e-9 relative on theta >= 1e-7 (the reference's significance floor, EM.cpp:409)
and 1e-15 absolute below it.
"""
import numpy as np
import pytest

import synth

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-9, 1e-15


def _check_theta(a, b):
    big = b >= 1e-7
    assert np.all(np.abs(a[big] - b[big]) <= RTOL * b[big])
    assert np.all(np.abs(a[~big] - b[~big]) <= ATOL + RTOL * b[~big])


@pytest.fixture(scope="module")
def ctx(built):
    import rsem_b200
    c = rsem_b200.Context(0)
    yield c
    c.close()


CASES = [
    # N, M, avg_deg, zipf, family, zero_rows
    (1, 5, 3, False, True, 0.0),
    (37, 50, 1, False, True, 0.0),
    (5000, 300, 5, False, True, 0.0),
    (20000, 5000, 10, False, True, 0.0),
    (20000, 5000, 20, False, False, 0.0),
    (30000, 2000, 6, True, True, 0.0),
    (30000, 2000, 40, False, True, 0.0),
    (4000, 400, 3, False, True, 0.3),
]


@pytest.mark.parametrize("variant", [0, 2, 4, 5])
@pytest.mark.parametrize("case", CASES)
def test_em_rounds_match_oracle(ctx, oracle, case, variant):
    N, M, deg, zipf, family, zero_rows = case
    row_ptr, sid, conprb, ncpv = synth.random_matrix(N, M, deg, seed=N + M, zipf=zipf, family=family, zero_rows=zero_rows)
    n0 = N / 20
    theta0 = synth.init_theta(M, n0, N + n0)
    from rsem_b200 import RsemB200Error
    for unknown in (1, 3, 6, -1):
        with pytest.raises(RsemB200Error):
            ctx.set_estep_variant(unknown)
    ctx.set_estep_variant(variant)
    ctx.upload_hits(row_ptr, sid, M)
    ctx.upload_conprb(conprb, ncpv)
    ctx.set_theta(theta0)
    if zero_rows > 0 and variant == 4:
        # rows without hits are legal at the C ABI but never produced by rsem-parse-alignments; the class layout
        # (variants 0 / 5) and the direct kernel handle them, asking for the staged row kernel must fail loudly
        with pytest.raises(RsemB200Error):
            ctx.em_rounds(1, 7, 20, 10000, n0)
        return
    stats, stopped = ctx.em_rounds(1, 7, 20, 10000, n0)
    theta_ref, stats_ref, _ = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 1, 7, 20, 10000)
    assert len(stats) == 7 and not stopped
    _check_theta(ctx.get_theta(), theta_ref)
    for (s, b, t), (s2, b2, t2) in zip(stats, stats_ref):
        assert abs(s - s2) <= 1e-9 * s2
        assert abs(b - b2) <= 1e-6 * b2 + 1e-12
        assert abs(t - t2) <= 2  # a change sitting exactly on the 1e-3 threshold may flip


def test_stop_condition_on_device(ctx, oracle):
    """the loop condition ROUND < MIN || (totNum > 0 && ROUND < MAX) is evaluated on the device"""
    row_ptr, sid, conprb, ncpv = synth.random_matrix(3000, 40, 2, seed=5, tiny_frac=0, family=False)
    n0 = 100.0
    theta0 = synth.init_theta(40, n0, 3100)
    ctx.set_estep_variant(0)
    ctx.upload_hits(row_ptr, sid, 40)
    ctx.upload_conprb(conprb, ncpv)
    ctx.set_theta(theta0)
    stats, stopped = ctx.em_rounds(1, 400, 5, 300, n0)
    theta_ref, stats_ref, stopped_ref = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 1, 400, 5, 300)
    assert stopped and stopped_ref
    assert len(stats) == len(stats_ref)
    _check_theta(ctx.get_theta(), theta_ref)


def test_expected_weights(ctx, oracle):
    row_ptr, sid, conprb, ncpv = synth.random_matrix(8000, 700, 8, seed=9)
    theta = np.random.default_rng(1).random(701)
    theta /= theta.sum()
    for variant in (0, 2, 4):
        ctx.set_estep_variant(variant)
        ctx.upload_hits(row_ptr, sid, 700)
        ctx.upload_conprb(conprb, ncpv)
        ctx.set_theta(theta)
        counts = ctx.expected_weights()
        post, post0 = ctx.download_conprb()
        c_ref, p_ref, p0_ref = oracle.estep(row_ptr, sid, conprb, ncpv, theta, want_post=True)
        assert np.allclose(counts, c_ref, rtol=1e-10, atol=1e-13)
        assert np.allclose(post, p_ref, rtol=1e-12, atol=0)
        assert np.allclose(post0, p0_ref, rtol=1e-12, atol=0)


def test_all_rows_below_epsilon(ctx):
    """rows whose sum < 1e-300 contribute nothing (EM.cpp:223); with N0 > 0 theta collapses to noise"""
    row_ptr = np.array([0, 2, 3], np.uint64)
    sid = np.array([1, -2, 2], np.int32)
    ctx.set_estep_variant(0)
    ctx.upload_hits(row_ptr, sid, 2)
    ctx.upload_conprb(np.array([1e-310, 0.0, 1e-305]), np.array([0.0, 1e-320]))
    ctx.set_theta(np.array([0.2, 0.4, 0.4]))
    stats, _ = ctx.em_rounds(1, 1, 20, 100, 3.0)
    assert stats[0][0] == 3.0
    assert np.array_equal(ctx.get_theta(), np.array([1.0, 0.0, 0.0]))


def test_rows_longer_than_a_stage_get_their_own_launch(ctx, oracle):
    """a 6000-hit row does not fit a shared-memory stage: the class layout leaves it to the long-row launch (frozen
    rounds), the posterior pass falls back to the unstaged kernel; both stay exact"""
    rng = np.random.default_rng(3)
    row_ptr, sid, conprb, ncpv = synth.random_matrix(3000, 8000, 7, seed=21)
    # splice one very long row into the middle
    long_deg = 6000
    mid = 1500
    h = int(row_ptr[mid])
    long_sid = (rng.permutation(8000)[:long_deg] + 1).astype(np.int32)
    long_con = 10.0 ** rng.uniform(-60, -3, size=long_deg)
    sid = np.concatenate([sid[:h], long_sid, sid[h:]])
    conprb = np.concatenate([conprb[:h], long_con, conprb[h:]])
    row_ptr = np.concatenate([row_ptr[:mid + 1], row_ptr[mid:] + np.uint64(long_deg)]).astype(np.uint64)
    ncpv = np.concatenate([ncpv[:mid], [1e-50], ncpv[mid:]])
    N, M = len(ncpv), 8000
    assert row_ptr[-1] == len(sid) and len(row_ptr) == N + 1
    n0 = 50.0
    theta0 = synth.init_theta(M, n0, N + n0)
    ctx.set_estep_variant(0)
    ctx.upload_hits(row_ptr, sid, M)
    ctx.upload_conprb(conprb, ncpv)
    ctx.set_theta(theta0)
    ctx.em_rounds(1, 5, 20, 10000, n0)
    theta_ref, _, _ = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 1, 5, 20, 10000)
    _check_theta(ctx.get_theta(), theta_ref)
    info = ctx.class_layout_info()
    assert info["built"] == 1 and info["long_rows"] == 1 and info["rows"] == N - 1
    counts = ctx.expected_weights()
    c_ref, _, _ = oracle.estep(row_ptr, sid, conprb, ncpv, ctx.get_theta(), want_post=True)
    assert np.allclose(counts, c_ref, rtol=1e-10, atol=1e-13)


def _class_matrix(N, M, deg, seed, dup, zipf=False):
    """rows drawn from a pool of N / dup distinct transcript lists (equivalence classes of ~dup reads), shuffled,
    with independent conprb per read - the structure the class layout exploits"""
    rng = np.random.default_rng(seed)
    pool_rp, pool_sid, _, _ = synth.random_matrix(max(1, N // dup), M, deg, seed=seed + 1, zipf=zipf)
    pool_rp = pool_rp.astype(np.int64)
    pick = rng.integers(0, len(pool_rp) - 1, size=N)
    degs = (pool_rp[pick + 1] - pool_rp[pick])
    row_ptr = np.zeros(N + 1, np.uint64)
    row_ptr[1:] = np.cumsum(degs)
    H = int(row_ptr[-1])
    src = np.repeat(pool_rp[pick], degs) + (np.arange(H) - np.repeat(row_ptr[:-1].astype(np.int64), degs))
    sid = np.abs(pool_sid[src]) * np.where(rng.random(H) < 0.5, 1, -1).astype(np.int32)  # strands differ inside a class
    conprb = 10.0 ** rng.uniform(-60, -3, size=H)
    conprb[rng.random(H) < 0.02] = 10.0 ** rng.uniform(-320, -295, size=1)
    conprb[rng.random(H) < 0.01] = 0.0
    ncpv = 10.0 ** rng.uniform(-80, -40, size=N)
    ncpv[rng.random(N) < 0.05] = 0.0
    return row_ptr, sid.astype(np.int32), conprb, ncpv


CLASS_CASES = [
    # N, M, deg, dup, zipf, rows per segment, CTA threads
    (40000, 3000, 20, 12, False, 8, 1024),     # C3-like: classes of ~12 reads
    (40000, 3000, 20, 12, False, 8, 512),
    (40000, 3000, 20, 200, False, 16, 1024),   # large classes: one-class batches, folded reductions
    (60000, 500, 2, 300, False, 8, 1024),      # degree <= 4: thread per segment
    (30000, 4000, 6, 1, False, 8, 1024),       # hardly any duplicates: segments of one row
    (30000, 3000, 40, 20, False, 3, 512),      # 16 lanes per segment, odd segment size
    (20000, 6000, 100, 10, False, 8, 1024),    # 32 lanes per segment
    (50000, 2000, 0, 30, True, 8, 1024),       # Zipf degrees 1..200 (C5 shape)
]


@pytest.mark.parametrize("case", CLASS_CASES)
def test_class_layout_matches_oracle(ctx, oracle, case, monkeypatch):
    """variant 5 (equivalence-class layout) on matrices with real class structure, every lane-group configuration"""
    N, M, deg, dup, zipf, seg_rows, threads = case
    monkeypatch.setenv("RSEM_B200_CLASS_ROWS", str(seg_rows))
    monkeypatch.setenv("RSEM_B200_CLASS_THREADS", str(threads))
    row_ptr, sid, conprb, ncpv = _class_matrix(N, M, deg, seed=N + deg, dup=dup, zipf=zipf)
    n0 = N / 20
    theta0 = synth.init_theta(M, n0, N + n0)
    ctx.set_estep_variant(5)
    ctx.upload_hits(row_ptr, sid, M)
    ctx.upload_conprb(conprb, ncpv)
    ctx.set_theta(theta0)
    stats, _ = ctx.em_rounds(1, 6, 20, 10000, n0)
    info = ctx.class_layout_info()
    assert info["built"] == 1 and info["rows"] == N and info["vals"] == int(row_ptr[-1]) + N
    if dup >= 10:
        assert info["segments"] < N / 2  # classes were found
    theta_ref, stats_ref, _ = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 1, 6, 20, 10000)
    _check_theta(ctx.get_theta(), theta_ref)
    for (s, b, t), (s2, b2, t2) in zip(stats, stats_ref):
        assert abs(s - s2) <= 1e-9 * s2
        assert abs(t - t2) <= 2
    # conprb changes (a model round in the executable): the value stream must be re-gathered
    conprb2 = conprb[::-1].copy()
    ctx.upload_conprb(conprb2, ncpv)
    ctx.set_theta(theta0)
    ctx.em_rounds(1, 3, 20, 10000, n0)
    theta_ref, _, _ = oracle.em_rounds(row_ptr, sid, conprb2, ncpv, theta0, n0, 1, 3, 20, 10000)
    _check_theta(ctx.get_theta(), theta_ref)
    ctx.set_estep_variant(0)


@pytest.mark.parametrize("threads", [512, 640, 1024])
def test_class_layout_ring_reuse(ctx, oracle, threads, monkeypatch):
    """enough tiles (~1600) that every persistent CTA refills its shared-memory stages several times: the producer /
    consumer hand-over of the ring is exercised, not only its first fill"""
    monkeypatch.setenv("RSEM_B200_CLASS_THREADS", str(threads))
    N, M = 500_000, 20_000
    row_ptr, sid, conprb, ncpv = _class_matrix(N, M, 20, seed=11, dup=10)
    n0 = N / 20
    theta0 = synth.init_theta(M, n0, N + n0)
    theta_ref, _, _ = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 1, 3, 20, 10000, n_threads=16)
    ctx.set_estep_variant(5)
    ctx.upload_hits(row_ptr, sid, M)
    ctx.upload_conprb(conprb, ncpv)
    for _ in range(5):  # repeated: a hand-over race would be timing dependent
        ctx.set_theta(theta0)
        ctx.em_rounds(1, 3, 20, 10000, n0)
        _check_theta(ctx.get_theta(), theta_ref)
    assert ctx.class_layout_info()["tiles"] > 3 * 148
    ctx.set_estep_variant(0)


def test_class_layout_c5_shape_one_million_reads(ctx, oracle):
    """BASELINE configs[4] shape at a size the oracle finishes in seconds: Zipf(1.1) degrees capped at 200, 1 M reads,
    every kernel variant against the oracle"""
    N, M = 1_000_000, 40_000
    row_ptr, sid, conprb, ncpv = _class_matrix(N, M, 0, seed=5, dup=25, zipf=True)
    n0 = N / 20
    theta0 = synth.init_theta(M, n0, N + n0)
    theta_ref, _, _ = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 1, 4, 20, 10000, n_threads=16)
    for variant in (5, 4, 2):
        ctx.set_estep_variant(variant)
        ctx.upload_hits(row_ptr, sid, M)
        ctx.upload_conprb(conprb, ncpv)
        ctx.set_theta(theta0)
        ctx.em_rounds(1, 4, 20, 10000, n0)
        _check_theta(ctx.get_theta(), theta_ref)
    ctx.set_estep_variant(0)


def test_row_group_kernel_ring_reuse(ctx, oracle):
    """enough tiles that every persistent CTA of the row kernel refills each of its three shared-memory stages at
    least twice: the hand-over of a stage from the warp that finishes it last to the next copy is exercised, in the
    frozen rounds (variant 4) and in the posterior pass"""
    N, M = 300_000, 20_000
    row_ptr, sid, conprb, ncpv = synth.random_matrix(N, M, 20, seed=12)
    # tiles of the row kernel (em_build_tiles): row r goes to tile (row_ptr[r] + r) // W, W = 4 * 1024 - 2 - max degree
    W = 4 * 1024 - 2 - int(np.diff(row_ptr.astype(np.int64)).max())
    n_tiles = len(np.unique((row_ptr[:-1].astype(np.int64) + np.arange(N)) // W))
    assert n_tiles >= 3 * 3 * 148  # 3 stages, each filled >= 3 times, on up to 148 SMs
    n0 = N / 20
    theta0 = synth.init_theta(M, n0, N + n0)
    ctx.set_estep_variant(4)
    ctx.upload_hits(row_ptr, sid, M)
    ctx.upload_conprb(conprb, ncpv)
    ctx.set_theta(theta0)
    ctx.em_rounds(1, 6, 20, 10000, n0)
    theta_ref, _, _ = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 1, 6, 20, 10000, n_threads=16)
    _check_theta(ctx.get_theta(), theta_ref)
    counts = ctx.expected_weights()
    post, post0 = ctx.download_conprb()
    c_ref, p_ref, p0_ref = oracle.estep(row_ptr, sid, conprb, ncpv, ctx.get_theta(), want_post=True, n_threads=16)
    assert np.allclose(counts, c_ref, rtol=1e-10, atol=1e-13)
    assert np.allclose(post, p_ref, rtol=1e-12, atol=0)
    assert np.allclose(post0, p0_ref, rtol=1e-12, atol=0)
    ctx.set_estep_variant(0)


def test_full_size_properties(ctx):
    """BASELINE configs[2] (C3: 50 M reads x 200 k transcripts, 1e9 hits) is far beyond what the CPU oracle finishes
    in seconds, so the full size is checked through properties that do not depend on it:
      * theta sums to 1 and the expected counts sum to the number of reads (every row has a positive sum);
      * scaling every conprb / ncpv by 2^-20 (exact in fp64) leaves the posteriors, hence theta, unchanged;
      * a prefix of the matrix goes through the small-size upload path that the oracle tests cover."""
    torch = pytest.importorskip("torch")
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
    import bench
    free, _ = torch.cuda.mem_get_info()
    if free < 60e9:
        pytest.skip("needs ~45 GB of free device memory")
    dev = torch.device("cuda:0")
    N, M, deg = 50_000_000, 200_000, 20
    row_ptr, sid, conprb, ncpv, H = bench.gen_matrix_torch(torch, dev, N, M, deg, seed=77)
    n0 = N / 20
    theta0 = synth.init_theta(M, n0, N + n0)
    ctx.set_estep_variant(0)
    torch.cuda.synchronize()  # the generator's stream is not the context's
    ctx.adopt_device_matrix(N, H, M, row_ptr.data_ptr(), sid.data_ptr(), conprb.data_ptr(), ncpv.data_ptr())
    ctx.set_theta(theta0)
    stats, _ = ctx.em_rounds(1, 3, 20, 10000, n0)
    th_a = ctx.get_theta()
    assert abs(th_a.sum() - 1.0) < 1e-12
    for s, _, _ in stats:
        assert abs(s - (N + n0)) <= 1e-9 * (N + n0)  # sum of counts + N0: every read distributes exactly one unit
    # exact power-of-two rescaling
    conprb.mul_(2.0 ** -20)
    ncpv.mul_(2.0 ** -20)
    torch.cuda.synchronize()
    ctx.adopt_device_matrix(N, H, M, row_ptr.data_ptr(), sid.data_ptr(), conprb.data_ptr(), ncpv.data_ptr())
    ctx.set_theta(theta0)
    ctx.em_rounds(1, 3, 20, 10000, n0)
    th_b = ctx.get_theta()
    big = th_a >= 1e-7
    assert np.all(np.abs(th_a[big] - th_b[big]) <= 1e-11 * th_a[big])
    # a prefix of the same matrix through the small-size (oracle-checked) upload path: one unit per read again
    n_sub = 100_000
    h_sub = int(row_ptr[n_sub].item())
    rp = row_ptr[: n_sub + 1].cpu().numpy().astype(np.uint64)
    sd = sid[:h_sub].cpu().numpy()
    cp = conprb[:h_sub].cpu().numpy()
    nc = ncpv[:n_sub].cpu().numpy()
    ctx.upload_hits(rp, sd, M)  # releases the adopted pointers before the tensors go away
    ctx.upload_conprb(cp, nc)
    del row_ptr, sid, conprb, ncpv
    torch.cuda.empty_cache()
    ctx.set_theta(th_a)
    counts_sub = ctx.expected_weights()
    assert abs(counts_sub.sum() - n_sub) <= 1e-9 * n_sub
