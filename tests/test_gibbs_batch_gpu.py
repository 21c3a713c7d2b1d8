"""K13 (rsem_b200_gibbs_batch_*) against the single-sample path and the CPU oracle: several samples in one batch, and for
every (sample, chain) job the count vectors and the chain_acc block bit-identical to Context.gibbs_run_chains on that sample
alone, the count vectors equal to oracle.gibbs_chain.  The matrices are test_gibbs_gpu's builders."""
import ctypes as C

import numpy as np
import pytest

from rsem_b200.capi import (GIBBS_BATCH_MAX_READS, GIBBS_BATCH_MIN_READS, RSEM_B200_ERR_ARG, RSEM_B200_ERR_FULL,
                            RSEM_B200_ERR_UNSUPPORTED, GibbsBatch, GibbsParams, RsemB200Error)
from test_gibbs_gpu import (Problem, _components, _csr, _family_matrix, _lane_matrix, _ofg_like, _rows, _to_rows,
                            _with_omitted, ctx)  # noqa: F401  (ctx: the module's context fixture)

pytestmark = pytest.mark.gpu

M = 300   # every sample of a batch has the reference's M


class Case:
    """a Problem with its chains: samples per chain, seeds, burn-in, gap"""

    def __init__(self, pb, samples, seeds, burnin, gap):
        self.pb, self.burnin, self.gap = pb, burnin, gap
        self.samples = np.ascontiguousarray(samples, np.int32)
        self.seeds = np.ascontiguousarray(seeds, np.uint32)
        self.keep = [np.ascontiguousarray(x, t) for x, t in ((pb.init, np.int32), (pb.alpha, np.float64), (pb.eel, np.float64),
                                                              (pb.mw, np.float64), (pb.genes, np.int32))]

    def params(self):
        init, alpha, eel, mw, genes = self.keep
        p = GibbsParams()
        p.M, p.burnin, p.gap, p.n_chains = self.pb.M, self.burnin, self.gap, len(self.samples)
        p.chain_samples = self.samples.ctypes.data_as(C.POINTER(C.c_int32))
        p.chain_seeds = self.seeds.ctypes.data_as(C.POINTER(C.c_uint32))
        p.n0, p.totc = self.pb.n0, self.pb.totc
        p.init_counts = init.ctypes.data_as(C.POINTER(C.c_int32))
        p.pseudo_counts = alpha.ctypes.data_as(C.POINTER(C.c_double))
        p.eel, p.mw = eel.ctypes.data_as(C.POINTER(C.c_double)), mw.ctypes.data_as(C.POINTER(C.c_double))
        p.n_genes = len(genes) - 1
        p.gene_start = genes.ctypes.data_as(C.POINTER(C.c_int32))
        return p

    def single(self, ctx):
        pb = self.pb
        ctx.gibbs_upload(pb.rp, pb.sid, pb.val, pb.M)
        cv = np.zeros((int(self.samples.sum()), pb.M + 1), np.int32)
        acc = np.zeros((len(self.samples), 4 * (pb.M + 1) + len(pb.genes) - 1))
        ctx.gibbs_run_chains(self.params(), cv, acc)
        return cv, acc


def _pb(rp, sid, val, seed, n0=100.0, **kw):
    return Problem(rp, sid, val, M, seed=seed, n0=n0, **kw)


def _run_batch(ctx, oracle, cases, worker_ctas=0, check_oracle=True):
    """all cases in one batch; every job against the single-sample path (bit for bit) and the oracle; -> batch stats"""
    with GibbsBatch(ctx, worker_ctas=worker_ctas) as b:
        slots = [b.add(c.pb.rp, c.pb.sid, c.pb.val, c.params()) for c in cases]
        st = b.run()
        assert st.jobs == sum(len(c.samples) for c in cases)
        assert st.worker_ctas == (worker_ctas or 2)
        outs = [b.result(s) for s in slots]
    for k, (c, (cv, acc)) in enumerate(zip(cases, outs)):
        cv1, acc1 = c.single(ctx)
        assert np.array_equal(cv, cv1), f"sample {k}: count vectors"
        assert np.array_equal(acc.view(np.uint64), acc1.view(np.uint64)), f"sample {k}: chain_acc"
        if check_oracle:
            at, pb = 0, c.pb
            for t, ns in enumerate(c.samples):
                ref, _ = oracle.gibbs_chain(pb.rp, pb.sid, pb.val, pb.M, pb.n0, pb.init, pb.alpha, pb.totc, pb.eel, pb.mw, pb.genes,
                                            c.burnin, c.gap, int(ns), int(c.seeds[t]))
                assert np.array_equal(cv[at:at + ns], ref), f"sample {k} chain {t}"
                at += ns
    return st


def _noise_only_rows(seed):
    rows = _to_rows(*_ofg_like(2000, M, 4, seed=seed, noise_scale=1.0))
    for i in range(0, len(rows), 40):
        rows[i] = ([0], [1e-8])
    return _csr(rows)


def _mixed_cases(oracle):
    cases = []
    # exactly 1248 reads, small families (counts in registers)
    rp, sid, val = _family_matrix(1248, M, seed=1, max_family=12, junk=0.02)
    assert len(rp) - 1 == GIBBS_BATCH_MIN_READS
    cases.append(Case(_pb(rp, sid, val, 1), [3, 3], oracle.chain_seeds(1, 2), 2, 1))
    # components of >= 32 transcripts (counts in L2); no burn-in, a gap of 3, chains of 1 and 4 samples (9 over 4 chains)
    rp, sid, val = _family_matrix(3000, M, seed=9, max_family=40, junk=0.3)
    assert _components(rp, sid, M)[0].max() >= 32
    cases.append(Case(_pb(rp, sid, val, 9), [3, 2, 2, 2], oracle.chain_seeds(9, 4), 0, 3))
    # omitted transcripts with per-transcript priors
    rp, sid, val, _, init = _with_omitted(5, 12)
    alpha = np.random.default_rng(5).uniform(0.05, 3.0, M + 1)
    alpha[init < 0] = 0.0
    cases.append(Case(_pb(rp, sid, val, 5, init=init, alpha=alpha), [2, 2, 1], oracle.chain_seeds(5, 3), 3, 2))
    # noise entries as heavy as the rest and a small noise count: many passes per sweep
    rp, sid, val = _ofg_like(3000, M, 4, seed=11, noise_scale=1.0)
    cases.append(Case(_pb(rp, sid, val, 11, n0=5.0), [2, 2], oracle.chain_seeds(11, 2), 4, 1))
    # rows holding only the noise entry
    rp, sid, val = _noise_only_rows(13)
    assert (_rows(rp) == 1).sum() >= 40
    cases.append(Case(_pb(rp, sid, val, 13), [2, 1], oracle.chain_seeds(13, 2), 2, 1))
    # rows longer than 16 and than 32 entries, families of 30 .. 33 transcripts
    rp, sid, val, _ = _lane_matrix(2500, 17)
    lens = _rows(rp)
    assert (lens > 16).any() and (lens > 32).any()
    cases.append(Case(_pb(rp, sid, val, 17), [2, 2], oracle.chain_seeds(17, 2), 2, 1))
    return cases


@pytest.mark.parametrize("worker_ctas", [1, 2, 3])
def test_samples_match_single_and_oracle(ctx, oracle, worker_ctas):
    _run_batch(ctx, oracle, _mixed_cases(oracle), worker_ctas)


def test_more_jobs_than_teams(ctx, oracle):
    """48 samples x 8 chains with one worker CTA per team: more jobs than co-resident teams, so teams claim again"""
    cases = []
    for s in range(48):
        rp, sid, val = _family_matrix(1300 + 7 * s, M, seed=100 + s, max_family=12, junk=0.1)
        cases.append(Case(_pb(rp, sid, val, 100 + s), [1] * 7 + [2], oracle.chain_seeds(100 + s, 8), 1, 1))
    st = _run_batch(ctx, oracle, cases, worker_ctas=1, check_oracle=False)
    assert st.jobs > st.teams
    _run_batch(ctx, oracle, cases[:3], worker_ctas=1)   # the oracle on a few of them


def test_single_job(ctx, oracle):
    rp, sid, val = _family_matrix(2000, M, seed=21, max_family=20, junk=0.05)
    st = _run_batch(ctx, oracle, [Case(_pb(rp, sid, val, 21), [3], oracle.chain_seeds(21, 1), 2, 1)])
    assert st.jobs == 1 and st.teams == 1


def test_arena_full_then_clear(ctx, oracle):
    """a capacity of one sample: the second add is refused with ERR_FULL; after a run and clear it fits"""
    cases = _mixed_cases(oracle)[:2]
    with GibbsBatch(ctx) as probe:
        need = probe.sample_bytes(len(cases[0].pb.rp) - 1, len(cases[0].pb.sid), M, len(cases[0].pb.genes) - 1,
                                  int(cases[0].samples.sum()), len(cases[0].samples))
    with GibbsBatch(ctx, capacity_bytes=need) as b:
        s0 = b.add(cases[0].pb.rp, cases[0].pb.sid, cases[0].pb.val, cases[0].params())
        with pytest.raises(RsemB200Error) as e:
            b.add(cases[1].pb.rp, cases[1].pb.sid, cases[1].pb.val, cases[1].params())
        assert e.value.code == RSEM_B200_ERR_FULL
        b.run()
        cv, _ = b.result(s0)
        assert np.array_equal(cv, cases[0].single(ctx)[0])
        b.clear()
        b.add(cases[0].pb.rp, cases[0].pb.sid, cases[0].pb.val, cases[0].params())


def test_refusals(ctx, oracle):
    with GibbsBatch(ctx) as b:
        for n1 in (GIBBS_BATCH_MIN_READS - 1, GIBBS_BATCH_MAX_READS + 1):   # the size rule
            with pytest.raises(RsemB200Error) as e:
                b.sample_bytes(n1, 4 * n1, M, 100, 8, 8)
            assert "size rule" in str(e.value)
        rp, sid, val = _ofg_like(1000, M, 4, seed=3, noise_scale=1.0)
        with pytest.raises(RsemB200Error) as e:
            b.add(rp, sid, val, Case(_pb(rp, sid, val, 3), [2], [7], 1, 1).params())
        assert e.value.code == RSEM_B200_ERR_UNSUPPORTED
        rows = _to_rows(*_ofg_like(2000, M, 4, seed=4, noise_scale=1.0))
        rows[1000] = ([], [])
        rp, sid, val = _csr(rows)
        with pytest.raises(RsemB200Error) as e:
            b.add(rp, sid, val, Case(_pb(rp, sid, val, 4), [2], [7], 1, 1).params())
        assert e.value.code == RSEM_B200_ERR_ARG and "a read without any entry" in str(e.value)
        assert b.run().jobs == 0
