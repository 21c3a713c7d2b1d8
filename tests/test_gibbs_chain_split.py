"""CPU checks of the host arithmetic behind a Gibbs run spread over several GPUs: the chain split
(rsem_b200_gibbs_split_chains) and the chain-order sum of the per-chain blocks (rsem_b200_gibbs_sum_chains).  Neither
needs a device."""
import ctypes as C

import numpy as np
import pytest

import rsem_b200
from rsem_b200.capi import GibbsOut, GibbsParams, RsemB200Error


def _lib():
    return rsem_b200.load_library()


def _samples(nsamples, chains):
    q, r = divmod(nsamples, chains)   # rsem-run-gibbs's split of NSAMPLES over the chains (Gibbs.cpp:211-223)
    return [q + (1 if i < r else 0) for i in range(chains)]


def _best_max(sweeps, parts):
    """smallest possible largest part over every contiguous split into `parts` non-empty ranges (brute force)"""
    n = len(sweeps)
    pre = np.concatenate([[0], np.cumsum(sweeps)])
    best = [[np.inf] * (n + 1) for _ in range(parts + 1)]
    best[0][0] = 0
    for k in range(1, parts + 1):
        for j in range(k, n + 1):
            best[k][j] = min(max(best[k - 1][i], pre[j] - pre[i]) for i in range(k - 1, j))
    return best[parts][n]


@pytest.mark.parametrize("nsamples,chains", [(7, 1), (10, 2), (10, 3), (20, 8), (1000, 9), (13, 13), (5, 4)])
@pytest.mark.parametrize("parts", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("burnin,gap", [(200, 1), (0, 1), (20, 7)])
def test_split_is_contiguous_and_balanced(nsamples, chains, parts, burnin, gap):
    samples = _samples(nsamples, chains)
    got = _lib().gibbs_split_chains(samples, burnin, gap, parts)
    used = min(parts, chains)
    assert got[0][0] == 0 and got[used - 1][1] == chains
    assert all(a < b for a, b in got[:used])                       # every used part has a chain
    assert all(got[i][1] == got[i + 1][0] for i in range(used - 1))  # contiguous, in chain order
    assert all(p == (chains, chains) for p in got[used:])          # the surplus parts are empty
    sweeps = [burnin + 1 + (s - 1) * gap for s in samples]
    loads = [sum(sweeps[a:b]) for a, b in got[:used]]
    # sweeps of the chains differ by at most one gap: the split is within one chain of the best one
    assert max(loads) <= _best_max(sweeps, used) + max(sweeps)
    assert got == _lib().gibbs_split_chains(samples, burnin, gap, parts)


def test_split_examples():
    lib = _lib()
    assert lib.gibbs_split_chains([5] * 8, 10, 1, 3) == [(0, 3), (3, 5), (5, 8)]   # targets 2.67 and 5.33 chains
    assert lib.gibbs_split_chains([2, 1], 0, 1, 2) == [(0, 1), (1, 2)]
    # one long chain and many short ones: the long one gets a device of its own
    assert lib.gibbs_split_chains([100, 1, 1, 1, 1], 0, 1, 2) == [(0, 1), (1, 5)]
    assert lib.gibbs_split_chains([3, 3, 3, 3], 0, 1, 3) == [(0, 1), (1, 3), (3, 4)]   # 1.33 -> 1, 2.67 -> 3
    assert lib.gibbs_split_chains([1, 2, 1], 0, 1, 2) == [(0, 1), (1, 3)]   # sweeps 1 2 1: 2 is as near 1 as 3: the lower


@pytest.mark.parametrize("bad", [dict(n_parts=0), dict(gap=0), dict(burnin=-1), dict(samples=[2, 0, 2])])
def test_split_refusals(bad):
    samples = bad.get("samples", [2, 2, 2])
    with pytest.raises(RsemB200Error):
        _lib().gibbs_split_chains(samples, bad.get("burnin", 1), bad.get("gap", 1), bad.get("n_parts", 2))


@pytest.mark.parametrize("chains,M,genes", [(1, 5, 2), (3, 40, 11), (9, 200, 0)])
def test_sum_in_chain_order(chains, M, genes):
    """the sums are the blocks added up from chain 0 on, in floating point (not a reassociated sum)"""
    rng = np.random.default_rng(chains)
    per = 4 * (M + 1) + genes
    acc = rng.standard_normal((chains, per)) * 10.0 ** rng.integers(-8, 9, (chains, per))
    p = GibbsParams()
    p.M, p.n_chains, p.n_genes = M, chains, genes
    sums = [np.full(M + 1, np.nan) for _ in range(4)] + [np.full(max(genes, 1), np.nan)]
    o = GibbsOut()
    o.sum_c, o.sum_c2, o.sum_tpm, o.sum_fpkm, o.sum_gene_c2 = (s.ctypes.data_as(C.POINTER(C.c_double)) for s in sums)
    _lib().gibbs_sum_chains(p, acc, o)
    want = np.zeros(per)
    for t in range(chains):
        want = want + acc[t]
    got = np.concatenate(sums[:4] + [sums[4][:genes]])
    assert np.array_equal(got, want)
