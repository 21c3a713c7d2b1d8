"""K13 (rsem_b200_gibbs_batch_*) at the edges of its team shape, team scratch, size rule and API, with test_gibbs_batch_gpu's
check: every (sample, chain) job bit-identical to Context.gibbs_run_chains on that sample alone (count vectors and the
chain_acc block), and equal to oracle.gibbs_chain (on a few samples where the batch is large).

Each case asserts the edge it is about: worker CTAs and teams from the launch's stats, against the rule of gibbs_batch_run
(teams = min(jobs, co-resident CTAs / (k + 1))); the claim order of the jobs, restated from gibbs_batch_run (reads x sweeps
of the chain, largest first); N1 and the flip-word count W = ceil(N1 / 32) from the CSR; components from the read x
transcript graph."""
import math

import numpy as np
import pytest

from rsem_b200.capi import (GIBBS_BATCH_MAX_READS, GIBBS_BATCH_MIN_READS, RSEM_B200_ERR_ARG, RSEM_B200_ERR_UNSUPPORTED,
                            GibbsBatch, RsemB200Error)
from test_gibbs_batch_gpu import M, Case, _mixed_cases, _pb, _run_batch
from test_gibbs_gpu import Problem, _components, _family_matrix, _ofg_like, ctx  # noqa: F401  (ctx: the module's context fixture)

pytestmark = pytest.mark.gpu

MAX_WORKERS = 8   # kBatchMaxWorkers


def _sweeps(c, t):
    """sweeps of chain t of a case: burn-in, then a kept draw every GAP sweeps (gibbs_batch_run's cost factor)"""
    return c.burnin + 2 + (int(c.samples[t]) - 1) * c.gap


def claim_order(cases):
    """the jobs (sample, chain) in the order teams claim them: N1 x sweeps, largest first, ties in add order"""
    jobs = [(r, t) for r, c in enumerate(cases) for t in range(len(c.samples))]
    return sorted(jobs, key=lambda j: -(len(cases[j[0]].pb.rp) - 1) * _sweeps(cases[j[0]], j[1]))


def _n1(c):
    return len(c.pb.rp) - 1


def _big_matrix(N1, seed):
    """N1 reads of 1..4 consecutive transcripts of M after the noise entry, built without a loop over the reads"""
    rng = np.random.default_rng(seed)
    deg = rng.integers(1, 5, N1)
    start = rng.integers(1, M - deg + 2)
    rp = np.zeros(N1 + 1, np.uint64)
    rp[1:] = np.cumsum(deg + 1)
    E = int(rp[-1])
    within = np.arange(E) - np.repeat(rp[:-1].astype(np.int64), deg + 1)
    sid = np.where(within == 0, 0, np.repeat(start, deg + 1) + within - 1).astype(np.int32)
    val = 10.0 ** rng.uniform(-12, -3, E)
    val[within == 0] = 10.0 ** rng.uniform(-14, -6, N1)
    return rp, sid, val


@pytest.fixture(scope="module")
def resident(ctx, oracle):
    """co-resident CTAs of gibbs_batch_kernel on this device (blocks per SM x SMs): 800 one-draw jobs with one worker CTA
    per team are more jobs than teams, so that launch has resident / 2 teams"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cases = []
    for s in range(8):
        rp, sid, val = _family_matrix(GIBBS_BATCH_MIN_READS + 40 * s, M, seed=300 + s, max_family=12, junk=0.1)
        cases.append(Case(_pb(rp, sid, val, 300 + s), [1] * 100, oracle.chain_seeds(300 + s, 100), 0, 1))
    st = _run_batch(ctx, oracle, cases, worker_ctas=1, check_oracle=False)
    assert st.jobs == 800 and st.jobs > st.teams
    per_sm = [p for p in range(1, 33) if p * sms // 2 == st.teams]
    assert len(per_sm) == 1
    return per_sm[0] * sms


# ---- 5. worker CTAs per team -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [4, 5, 8])
def test_worker_ctas_per_team(ctx, oracle, resident, k):
    """k = 4, 5 and kBatchMaxWorkers = 8 worker CTAs per team (the size of each job's slice totals) on the mixed samples plus
    one sample that is a single giant component, walked by all k workers"""
    rp, sid, val = _ofg_like(4000, M, 6, seed=31, noise_scale=1.0)
    ntr, _ = _components(rp, sid, M)
    assert ntr.max() >= 0.9 * M and (ntr == ntr.max()).mean() >= 0.9   # one component holds nearly every read
    cases = _mixed_cases(oracle) + [Case(_pb(rp, sid, val, 31), [2, 2, 1], oracle.chain_seeds(31, 3), 2, 1)]
    st = _run_batch(ctx, oracle, cases, worker_ctas=k)
    assert st.worker_ctas == k and st.teams == min(st.jobs, resident // (k + 1))


def test_nine_worker_ctas_refused(ctx):
    with pytest.raises(RsemB200Error) as e:
        GibbsBatch(ctx, worker_ctas=MAX_WORKERS + 1)
    assert f"error {RSEM_B200_ERR_ARG}:" in str(e.value) and "worker_ctas" in str(e.value)


# ---- 6. team scratch reused across jobs ---------------------------------------------------------------------------------------
LARGE_N1 = (4097, 4095, 4096)   # N1 = 1, 31 and 0 (mod 32): a partial last flip word of 1 and 31 bits, and none
SMALL_N1 = (1281, 1279, 1280)


def _alternating_cases(oracle, n_pairs, chains):
    """pairs of samples, a large-N1 one with few sweeps and a small-N1 one with many, whose costs N1 x sweeps interleave:
    large(p) > small(p) > large(p + 1); every chain of a sample keeps 2 draws with GAP 1, so the burn-in sets the sweeps"""
    cases = []
    for p in range(n_pairs):
        nl, ns = LARGE_N1[p % 3], SMALL_N1[p % 3]
        sw_l = 4 + n_pairs - p
        hi, lo = nl * sw_l, LARGE_N1[(p + 1) % 3] * (sw_l - 1)
        sw_s = (hi + lo) // 2 // ns
        for n1, sw, seed in ((nl, sw_l, 2 * p), (ns, sw_s, 2 * p + 1)):
            rp, sid, val = _family_matrix(n1, M, seed=500 + seed, max_family=20, junk=0.3)
            cases.append(Case(_pb(rp, sid, val, 500 + seed), [2] * chains, oracle.chain_seeds(500 + seed, chains), sw - 3, 1))
    return cases


def test_team_scratch_across_jobs(ctx, oracle, resident):
    """at least 4 x teams jobs whose claim order alternates between large-N1 / few-sweep samples and small-N1 / many-sweep
    samples: a team's z, uniforms, flips and prefix scratch (sized for the largest N1) go from a large job to a small one and
    back; N1 = 1, 31 and 0 (mod 32) on both sides"""
    k, chains = MAX_WORKERS, 6
    teams = resident // (k + 1)
    n_pairs = math.ceil(4 * teams / (2 * chains)) + 1
    cases = _alternating_cases(oracle, n_pairs, chains)
    order = claim_order(cases)
    n1 = [_n1(cases[r]) for r, _ in order]
    runs = [x for i, x in enumerate(n1) if i == 0 or x != n1[i - 1]]   # N1 along the claim order, repeats collapsed
    assert len(runs) == len(cases)                                     # every sample's jobs are claimed together ...
    assert all((x > 2000) == (i % 2 == 0) for i, x in enumerate(runs))  # ... and N1 falls, rises, falls, ... between them
    for side in (LARGE_N1, SMALL_N1):
        assert {x % 32 for x in side} == {0, 1, 31} and set(side) <= set(n1)
    st = _run_batch(ctx, oracle, cases, worker_ctas=k, check_oracle=False)
    assert st.teams == teams and st.jobs >= 4 * st.teams
    _run_batch(ctx, oracle, cases[:2], worker_ctas=k)   # the oracle on one large and one small sample


# ---- 7. size rule -----------------------------------------------------------------------------------------------------------
def test_size_rule_edges(ctx, oracle):
    """N1 = 1249 (1 mod 32) and N1 = 2^19 (W = 16384 flip words, the team scratch at its largest) with a short chain, in one
    batch with small samples; add refuses N1 = 1247 and 2^19 + 1 with ERR_UNSUPPORTED"""
    rp_lo, sid_lo, val_lo = _family_matrix(GIBBS_BATCH_MIN_READS + 1, M, seed=61, max_family=12, junk=0.3)
    rp_hi, sid_hi, val_hi = _big_matrix(GIBBS_BATCH_MAX_READS, seed=62)
    assert len(rp_lo) - 1 == 1249 and 1249 % 32 == 1
    assert len(rp_hi) - 1 == 1 << 19 and math.ceil((len(rp_hi) - 1) / 32) == 16384
    cases = [Case(_pb(rp_lo, sid_lo, val_lo, 61), [2, 3], oracle.chain_seeds(61, 2), 2, 1),
             Case(_pb(rp_hi, sid_hi, val_hi, 62), [2, 2], oracle.chain_seeds(62, 2), 0, 1)]
    cases += _mixed_cases(oracle)[:2]
    _run_batch(ctx, oracle, cases, worker_ctas=2)
    with GibbsBatch(ctx) as b:
        for n1, mk in ((GIBBS_BATCH_MIN_READS - 1, lambda n, s: _family_matrix(n, M, seed=s, max_family=12, junk=0.3)),
                       (GIBBS_BATCH_MAX_READS + 1, _big_matrix)):
            rp, sid, val = mk(n1, 63)
            assert len(rp) - 1 == n1
            with pytest.raises(RsemB200Error) as e:
                b.add(rp, sid, val, Case(_pb(rp, sid, val, 63), [2], [7], 0, 1).params())
            assert e.value.code == RSEM_B200_ERR_UNSUPPORTED and "size rule" in str(e.value)
        assert b.run().jobs == 0


# ---- 8. API paths -----------------------------------------------------------------------------------------------------------
def _same_as_single(ctx, c, out):
    cv, acc = out
    cv1, acc1 = c.single(ctx)
    assert np.array_equal(cv, cv1) and np.array_equal(acc.view(np.uint64), acc1.view(np.uint64))


def test_api_paths(ctx, oracle):
    """run -> add -> run without clear runs only the new slot and leaves the first results as they were; result before a
    run is refused; an add with another M or n_genes, or with a chain that keeps no draw, is refused; after clear the batch
    takes a new M"""
    a, b_, c_ = _mixed_cases(oracle)[:3]
    with GibbsBatch(ctx) as b:
        s_a = b.add(a.pb.rp, a.pb.sid, a.pb.val, a.params())
        assert b.run().jobs == len(a.samples)
        first = b.result(s_a)
        s_b = b.add(b_.pb.rp, b_.pb.sid, b_.pb.val, b_.params())
        with pytest.raises(RsemB200Error) as e:
            b.result(s_b)
        assert "has not run yet" in str(e.value)
        assert b.run().jobs == len(b_.samples)
        again = b.result(s_a)
        assert np.array_equal(first[0], again[0]) and np.array_equal(first[1].view(np.uint64), again[1].view(np.uint64))
        _same_as_single(ctx, a, again)
        _same_as_single(ctx, b_, b.result(s_b))
        assert b.run().jobs == 0

        rp, sid, val = _family_matrix(2000, 250, seed=71, max_family=12, junk=0.1)
        other_m = Case(Problem(rp, sid, val, 250, seed=71), [2], oracle.chain_seeds(71, 1), 1, 1)
        pb = _pb(c_.pb.rp, c_.pb.sid, c_.pb.val, 72)
        pb.genes = np.append(np.arange(1, M + 1, 2, dtype=np.int32), np.int32(M + 1))
        assert len(pb.genes) - 1 != len(a.pb.genes) - 1
        other_genes = Case(pb, [2], oracle.chain_seeds(72, 1), 1, 1)
        no_draw = Case(_pb(c_.pb.rp, c_.pb.sid, c_.pb.val, 73), [2, 0], oracle.chain_seeds(73, 2), 1, 1)
        for bad, why in ((other_m, "the M and n_genes of the first"), (other_genes, "the M and n_genes of the first"),
                         (no_draw, "at least one sample")):
            with pytest.raises(RsemB200Error) as e:
                b.add(bad.pb.rp, bad.pb.sid, bad.pb.val, bad.params())
            assert e.value.code == RSEM_B200_ERR_ARG and why in str(e.value)

        b.clear()
        s = b.add(other_m.pb.rp, other_m.pb.sid, other_m.pb.val, other_m.params())
        assert b.run().jobs == 1
        out = b.result(s)
        _same_as_single(ctx, other_m, out)
        pb = other_m.pb
        ref, _ = oracle.gibbs_chain(pb.rp, pb.sid, pb.val, pb.M, pb.n0, pb.init, pb.alpha, pb.totc, pb.eel, pb.mw, pb.genes,
                                    1, 1, 2, int(other_m.seeds[0]))
        assert np.array_equal(out[0], ref)
