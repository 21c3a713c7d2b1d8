"""K12 (the batched frozen-conprb rounds, rsem_b200_batch_*) against the CPU oracle on each sample's full-M matrix.

Every sample runs round 1 on the oracle (after it theta is 0 for each transcript without a hit), is added to a batch
from round 2 on, and its per-round statistics, stop round, final theta and final-pass counts / posteriors are
compared with oracle.em_rounds / oracle.estep from the same theta.  Tolerances are those of test_em_kernels_gpu.py.
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


def _check_stats(stats, ref):
    assert len(stats) == len(ref)
    for (s, b, t), (s2, b2, t2) in zip(stats, ref):
        assert abs(s - s2) <= 1e-9 * s2
        assert abs(b - b2) <= 1e-6 * b2 + 1e-12
        assert abs(t - t2) <= 2  # a change sitting exactly on the 1e-3 threshold may flip


@pytest.fixture(scope="module")
def ctx(built):
    import rsem_b200
    c = rsem_b200.Context(0)
    yield c
    c.close()


def _sample(oracle, N, M, deg, seed, n0=None, **kw):
    row_ptr, sid, conprb, ncpv = synth.random_matrix(N, M, deg, seed=seed, **kw)
    n0 = N / 20 if n0 is None else n0
    theta0 = synth.init_theta(M, n0, N + n0)
    theta1, _, _ = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 1, 1, 20, 10000)
    return dict(m=(row_ptr, sid, conprb, ncpv), theta=theta1, n0=n0)


def _run_to_end(batch, slots, k):
    """launches of k rounds until every slot stopped: {slot: (stats, launches until it stopped)}"""
    out = {s: [] for s in slots}
    when = {}
    for launch in range(100000):
        res = batch.run(k)
        for s in slots:
            st, stopped = res[s]
            out[s] += st
            if stopped and s not in when:
                when[s] = launch
        if len(when) == len(slots):
            return {s: (out[s], when[s]) for s in slots}
    raise AssertionError("the batch did not stop")


def _compare(oracle, batch, slot, smp, min_round, max_round, stats):
    row_ptr, sid, conprb, ncpv = smp["m"]
    theta_ref, stats_ref, stopped_ref = oracle.em_rounds(row_ptr, sid, conprb, ncpv, smp["theta"], smp["n0"], 2, 100000,
                                                         min_round, max_round)
    assert stopped_ref
    _check_stats(stats, stats_ref)
    theta, counts, post, post0 = batch.final(slot, posteriors=True)
    _check_theta(theta, theta_ref)
    c_ref, p_ref, p0_ref = oracle.estep(row_ptr, sid, conprb, ncpv, theta, want_post=True)
    assert np.allclose(counts, c_ref, rtol=1e-10, atol=1e-13)
    assert np.allclose(post, p_ref, rtol=1e-12, atol=0)
    assert np.allclose(post0, p0_ref, rtol=1e-12, atol=0)


def test_more_samples_than_resident_ctas(ctx, oracle):
    """300 samples of varied size: the claim counter runs past every resident CTA, rounds cross launch boundaries"""
    import rsem_b200
    rng = np.random.default_rng(7)
    smps = [_sample(oracle, int(rng.integers(1, 3000)), int(rng.integers(5, 400)), int(rng.integers(1, 12)), seed=i)
            for i in range(300)]
    with rsem_b200.Batch(ctx) as b:
        slots = [b.add(*s["m"], s["theta"], s["n0"], 2, 20, 150) for s in smps]
        res = _run_to_end(b, slots, 16)
        for s, smp in zip(slots, smps):
            _compare(oracle, b, s, smp, 20, 150, res[s][0])


def test_stop_rounds(ctx, oracle):
    """stops at MIN_ROUND, at MAX_ROUND and in the first round of a launch, each with its own round counter"""
    import rsem_b200
    fast = _sample(oracle, 2000, 40, 1, seed=3, family=False, tiny_frac=0)   # unique reads: converges at once
    slow = _sample(oracle, 4000, 300, 8, seed=4)
    edge = _sample(oracle, 3000, 200, 6, seed=5)
    k = 7
    with rsem_b200.Batch(ctx) as b:
        s_fast = b.add(*fast["m"], fast["theta"], fast["n0"], 2, 20, 10000)
        s_slow = b.add(*slow["m"], slow["theta"], slow["n0"], 2, 1, 4)       # still changing at round 4
        s_edge = b.add(*edge["m"], edge["theta"], edge["n0"], 2, 2 + k, 2 + k)   # rounds 2..8 in launch 0, 9 opens launch 1
        res = _run_to_end(b, [s_fast, s_slow, s_edge], k)
        assert len(res[s_fast][0]) == 20 - 1
        assert len(res[s_slow][0]) == 4 - 1 and res[s_slow][0][-1][2] > 0
        assert len(res[s_edge][0]) == k + 1 and res[s_edge][1] == 1
        _compare(oracle, b, s_fast, fast, 20, 10000, res[s_fast][0])
        _compare(oracle, b, s_slow, slow, 1, 4, res[s_slow][0])
        _compare(oracle, b, s_edge, edge, 2 + k, 2 + k, res[s_edge][0])


def test_clamped_rows_noise_only_rows_and_edges(ctx, oracle):
    """rows below 1e-300, rows with only the noise entry alive, ncpv = 0, N0 = 0, a one-read sample, a one-transcript
    compact set"""
    import rsem_b200
    smps = []
    a = _sample(oracle, 3000, 100, 4, seed=11, tiny_frac=0.3)           # many terms below 1e-300
    smps.append(a)
    row_ptr, sid, conprb, ncpv = synth.random_matrix(3000, 100, 4, seed=12)
    conprb = conprb.copy()
    dead = np.repeat(np.random.default_rng(1).random(3000) < 0.2, np.diff(row_ptr.astype(np.int64)))
    conprb[dead] = 0.0                                                   # noise-only rows
    ncpv = ncpv.copy()
    ncpv[::3] = 0.0                                                      # ncpv = 0
    theta0 = synth.init_theta(100, 150.0, 3150)
    smps.append(dict(m=(row_ptr, sid, conprb, ncpv), n0=150.0,
                     theta=oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, 150.0, 1, 1, 20, 10000)[0]))
    smps.append(_sample(oracle, 2000, 80, 3, seed=13, n0=0.0))          # N0 = 0
    one = (np.array([0, 3], np.uint64), np.array([4, -9, 2], np.int32), np.array([1e-4, 3e-5, 2e-6]), np.array([1e-7]))
    t0 = synth.init_theta(10, 1.0, 2.0)
    smps.append(dict(m=one, n0=1.0, theta=oracle.em_rounds(*one, t0, 1.0, 1, 1, 20, 10000)[0]))
    solo = (np.arange(51, dtype=np.uint64), np.full(50, 7, np.int32), np.full(50, 1e-3), np.full(50, 1e-6))
    t0 = synth.init_theta(30, 5.0, 55.0)
    smps.append(dict(m=solo, n0=5.0, theta=oracle.em_rounds(*solo, t0, 5.0, 1, 1, 20, 10000)[0]))
    with rsem_b200.Batch(ctx) as b:
        slots = [b.add(*s["m"], s["theta"], s["n0"], 2, 20, 400) for s in smps]
        res = _run_to_end(b, slots, 9)
        for s, smp in zip(slots, smps):
            _compare(oracle, b, s, smp, 20, 400, res[s][0])


def _wide(oracle, m, seed):
    """a sample whose hits name exactly m distinct transcripts out of M = 2 m"""
    rng = np.random.default_rng(seed)
    M = 2 * m
    names = rng.permutation(M)[:m] + 1
    N = m + 500
    deg = rng.integers(1, 4, size=N)
    row_ptr = np.zeros(N + 1, np.uint64)
    row_ptr[1:] = np.cumsum(deg)
    H = int(row_ptr[-1])
    sid = names[rng.integers(0, m, size=H)]
    sid[:m] = names                                                      # every name is used
    sid = (sid * np.where(rng.random(H) < 0.5, 1, -1)).astype(np.int32)
    conprb = 10.0 ** rng.uniform(-12, -3, size=H)
    ncpv = 10.0 ** rng.uniform(-14, -8, size=N)
    n0 = 20.0
    theta0 = synth.init_theta(M, n0, N + n0)
    theta1 = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 1, 1, 20, 10000)[0]
    return dict(m=(row_ptr, sid, conprb, ncpv), theta=theta1, n0=n0)


def test_layout_edges_and_refusals(ctx, oracle):
    """12287 distinct transcripts fit shared memory, 12288 do not; a 2048-hit read fits a tile, 2049 does not; a
    theta that is not 0 outside the compact set is refused; a full arena refuses with its own code"""
    import rsem_b200
    from rsem_b200.capi import RSEM_B200_ERR_FULL
    at = _wide(oracle, 12287, 1)
    with rsem_b200.Batch(ctx) as b:
        s = b.add(*at["m"], at["theta"], at["n0"], 2, 20, 60)
        res = _run_to_end(b, [s], 25)
        _compare(oracle, b, s, at, 20, 60, res[s][0])
        past = _wide(oracle, 12288, 2)
        with pytest.raises(rsem_b200.RsemB200Error) as e:
            b.add(*past["m"], past["theta"], past["n0"], 2, 20, 60)
        assert e.value.code == 4
        for d, ok in ((2048, True), (2049, False)):
            row_ptr = np.array([0, d, d + 1], np.uint64)
            assert (b.sample_bytes(row_ptr, d) > 0) if ok else True
            if not ok:
                with pytest.raises(rsem_b200.RsemB200Error):
                    b.sample_bytes(row_ptr, d)
        row_ptr, sid, conprb, ncpv = at["m"]
        theta = at["theta"].copy()
        unnamed = np.setdiff1d(np.arange(1, len(theta)), np.abs(sid))[0]
        theta[unnamed] = 1e-30
        with pytest.raises(rsem_b200.RsemB200Error) as e:
            b.add(row_ptr, sid, conprb, ncpv, theta, at["n0"], 2, 20, 60)
        assert e.value.code == 2
    small = _sample(oracle, 1000, 50, 3, seed=21)
    with rsem_b200.Batch(ctx, 1) as b:
        need = b.sample_bytes(small["m"][0], len(np.unique(np.abs(small["m"][1]))))
    with rsem_b200.Batch(ctx, 2 * need) as b:
        s1 = b.add(*small["m"], small["theta"], small["n0"], 2, 20, 100)
        s2 = b.add(*small["m"], small["theta"], small["n0"], 2, 20, 100)
        with pytest.raises(rsem_b200.RsemB200Error) as e:
            b.add(*small["m"], small["theta"], small["n0"], 2, 20, 100)
        assert e.value.code == RSEM_B200_ERR_FULL
        b.remove(s1)
        s3 = b.add(*small["m"], small["theta"], small["n0"], 2, 20, 100)
        res = _run_to_end(b, [s2, s3], 11)
        for s in (s2, s3):
            _compare(oracle, b, s, small, 20, 100, res[s][0])
