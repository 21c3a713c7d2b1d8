"""K12 (k12_kernel<FINAL>, batch_kernels.cu) bit for bit against the CPU oracle, at its lane-group, tile, clamp,
threshold and stop-rule edges.

The inputs are test_csr_estep_exact_gpu.py's exact ones: theta and conprb powers of two and every row summing to a
power of two, so every weight, count, sum, theta, bChange and totNum is the same in any summation order.  K12 forms a
weight as f * (1 / sum) where the reference divides; the two agree only while 1 / sum is exact, so `==` is asserted
only where every row sum is a power of two: round 1 from the builders' theta, the final pass run straight after `add`
on that theta, and the fixed-point matrices below, which stay dyadic in every round.  A row whose only term is exactly
1e-300 is where the two part: 1e-300 * (1 / 1e-300) = 1 - 2^-53 where the oracle gives 1.

Every input goes through compact(): batch_add refuses a theta that is not 0 on a transcript no hit names, which is
what the M-step leaves from round 2 on.  Each case asserts from its CSR, through lanes_per_row and cut_tiles as
test_batch_edges_gpu.py restates them, that it reaches the edge it is about; the CPU half checks the builders."""
import functools
from fractions import Fraction

import numpy as np
import pytest

from test_batch_edges_gpu import G_THRESHOLDS, HIT_CAP, ROW_CAP, _stage_degrees, lanes_per_row, tiles
from test_csr_estep_exact_gpu import (BELOW, EPS, _change, _eq, converged_matrix, exact_matrix, fill_degrees,
                                      single_hit_matrix, threshold_matrix)
from test_em_batch_gpu import _run_to_end, ctx  # noqa: F401  (ctx: the module's context fixture)

gpu = pytest.mark.gpu

THREADS, STAGES, THETA_CAP = 512, 2, 12288   # kThreads, kStages, kThetaCap
NOMINAL_SMS = 132                            # H100 SXM; the GPU test sizes its launch from the device's own count
FIRST = 11                                   # rsem-run-em-batch hands a sample to the batch at round 11
CHUNK = 64                                   # rounds per launch in rsem-run-em-batch
LONE = EPS * (1.0 / EPS)                     # K12's weight of a row whose only term is exactly 1e-300


# ------------------------------------------------------------------------------------------------------------------
# samples in the batch's compact space
# ------------------------------------------------------------------------------------------------------------------
def compact(sid, theta):
    """theta with 0 on every transcript no hit names"""
    named = np.zeros(len(theta), bool)
    named[0] = True
    named[np.abs(np.asarray(sid, np.int64))] = True
    return np.where(named, theta, 0.0)


class Sample:
    def __init__(self, row_ptr, sid, conprb, ncpv, theta, n0, **facts):
        self.m = (np.asarray(row_ptr, np.uint64), np.asarray(sid, np.int32), np.asarray(conprb, np.float64),
                  np.asarray(ncpv, np.float64))
        self.theta = compact(self.m[1], np.asarray(theta, np.float64))
        self.n0 = float(n0)
        self.__dict__.update(facts)

    @property
    def N(self):
        return len(self.m[0]) - 1

    @property
    def H(self):
        return int(self.m[0][-1])

    @property
    def m1(self):
        return len(np.unique(np.abs(self.m[1]))) + 1

    @property
    def G(self):
        return lanes_per_row(self.N, self.H)

    @property
    def tiles(self):
        return tiles(self.m[0])

    def add(self, b, first_round=FIRST, min_round=FIRST + 9, max_round=10000):
        return b.add(*self.m, self.theta, self.n0, first_round, min_round, max_round)


def from_exact(x, **facts):
    return Sample(*x.mat, x.theta, x.n0, edges=x.edges, clamp=x.clamp, n_regular=x.n_regular, **facts)


def _deg(smp):
    return np.diff(smp.m[0].astype(np.int64))


# ------------------------------------------------------------------------------------------------------------------
# 1. lane groups: mean degree at and just above each threshold, clamp rows at hit positions 0, 1, G and 2G
# ------------------------------------------------------------------------------------------------------------------
LANE_CASES = [(T, above) for T in G_THRESHOLDS for above in (0, 1)]


@functools.lru_cache(maxsize=None)
def lane_case(T, above):
    N = 2000
    H = (T - 1) * N + above
    G = lanes_per_row(N, H)
    pos = sorted({0, 1, G, 2 * G})
    clamp = [(k, p) for p in pos for k in ("keep", "drop")]
    clamp += [("noise_keep",), ("noise_drop",), ("all", 1), ("all", 3), ("all", 2 * G + 1)]
    c_deg = [max(s[1] + 1, 2) if s[0] in ("keep", "drop") else 1 if s[0].startswith("noise") else s[1] for s in clamp]
    fixed = [G - 1, G, G + 1, 2 * G + 1] * 3   # G - 1 = 0 for G = 1: a row with the noise term only
    degs = fill_degrees(N - len(clamp), H - sum(c_deg), 1, max(2 * T, 2 * G + 2), fixed, seed=31 * T + above)
    smp = from_exact(exact_matrix(degs, seed=17 * T + above, clamp=clamp), clamp_pos=pos)
    # the edges it claims
    g = (1, 2, 4, 8, 16)[G_THRESHOLDS.index(T)]
    assert (smp.N, smp.H, smp.G) == (N, H, 2 * g if above else g)
    deg = _deg(smp)
    for d in (G - 1, G, G + 1, 2 * G + 1):
        assert (deg[:smp.n_regular] == d).any()
    if G > 1:   # more rows in a tile than one pass of the 16 warps covers (G = 1: one pass is a whole tile)
        assert max(re - rs for rs, re, _, _, _ in smp.tiles) > (THREADS // 32) * (32 // G)
    return smp


def lone_epsilon_sample():
    """regular exact rows and one row whose only surviving term is exactly 1e-300, on a transcript of its own, next to
    a term just below it, with ncpv = 0"""
    x = exact_matrix(np.full(700, 3), seed=99)
    M = x.M + 1
    theta = np.r_[x.theta, 2.0 ** -6]
    t_below = 1 + int(np.abs(x.sid[0])) % x.M
    sid = np.r_[x.sid, [M, -t_below]].astype(np.int32)
    conprb = np.r_[x.conprb, EPS * 2.0 ** 6, BELOW / theta[t_below]]
    assert theta[M] * conprb[-2] == EPS and theta[t_below] * conprb[-1] < EPS
    row_ptr = np.r_[x.row_ptr, x.row_ptr[-1] + 2].astype(np.uint64)
    return Sample(row_ptr, sid, conprb, np.r_[x.ncpv, 0.0], theta, x.n0, lone=M, lone_hit=len(sid) - 2)


# ------------------------------------------------------------------------------------------------------------------
# 2. tiles and stage copies
# ------------------------------------------------------------------------------------------------------------------
TILE_CASES = ["one", "rows", "hits", "stage-G1", "stage-G32"]


def _closed_by(smp):
    """(tiles closed by the row cap, tiles closed by the hit cap); the last tile is closed by the sample's end"""
    deg = _deg(smp)
    ts = smp.tiles
    by_rows = [t for t in ts[:-1] if t[1] - t[0] == ROW_CAP and t[3] - t[2] + deg[t[1]] <= HIT_CAP]
    by_hits = [t for t in ts[:-1] if t[3] - t[2] + deg[t[1]] > HIT_CAP]
    return by_rows, by_hits


@functools.lru_cache(maxsize=None)
def tile_case(name):
    if name == "one":
        smp = from_exact(exact_matrix(np.full(300, 5), seed=41))
        assert len(smp.tiles) == 1
    elif name == "rows":       # 512, 512 and 276 one-hit rows: tiles closed by the row cap, 3 tiles
        smp = from_exact(exact_matrix(np.full(1300, 1), seed=42))
        by_rows, _ = _closed_by(smp)
        assert len(smp.tiles) == 3 and len(by_rows) == 2
    elif name == "hits":       # 256 rows of 8 hits fill a tile to exactly 2048 hits: 2 tiles (= kStages)
        smp = from_exact(exact_matrix(np.full(300, 8), seed=43))
        _, by_hits = _closed_by(smp)
        assert len(smp.tiles) == STAGES and by_hits[0][3] - by_hits[0][2] == HIT_CAP
    else:                      # test_batch_edges_gpu's largest copies of each Stage array, on exact values
        filler_deg, n_fill, G = (1, 6000, 1) if name == "stage-G1" else (200, 400, 32)
        smp = from_exact(exact_matrix(np.asarray(_stage_degrees(filler_deg, n_fill)), seed=44 + G))
        assert smp.G == G
        ts = smp.tiles
        alone = [t for t in ts if t[1] - t[0] == 1 and t[3] - t[2] == HIT_CAP]   # a 2048-hit row alone in its tile
        assert len(alone) == 2 and alone[1][2] % 4 == 3
        assert alone[1][4]["sid"] == 2052 and alone[1][4]["con"] == 2050
        rs, re, hs, he, c = next(t for t in ts if t[0] == 3)
        assert (re - rs, hs % 4, he - hs) == (ROW_CAP, 3, HIT_CAP)
        assert c == dict(sid=2052, con=2050, rp=516, ncp=514)
        for a in c:
            assert max(t[4][a] for t in ts) == c[a]
    return smp


# ------------------------------------------------------------------------------------------------------------------
# 3. the M-step: the strided loop's warps and lanes, m1 up to kThetaCap, the 0.001 and 1e-7 thresholds
# ------------------------------------------------------------------------------------------------------------------
M1_CASES = [2, 33, 512, 513, 1025, THETA_CAP]


def mstep_positions(m1):
    """compact indices for the round's largest change: one in each warp of the 512-thread loop (in its latest lap),
    lanes 0 and 31, and m1 - 1"""
    M = m1 - 1
    pos = set()
    for w in range(THREADS // 32):
        for lap in (2, 1, 0):
            i = THREADS * lap + 32 * w + (5 * w + 3) % 32
            if 1 <= i <= M:
                pos.add(i)
                break
    pos |= {i for i in (31, 32, THREADS + 31, 2 * THREADS, M) if 1 <= i <= M}
    return sorted(pos)


@functools.lru_cache(maxsize=None)
def mstep_case(m1):
    """one sample per position p: every transcript 1..m1 - 1 named by single-hit rows of weight 1 (twice at p), theta
    2^-20 except 2^-23 at p, so p has the round's largest change; the compact space is the full one"""
    M = m1 - 1
    pos = mstep_positions(m1)
    counts = np.ones(m1, np.int64)
    counts[0] = 0
    counts[pos] = 2
    base = np.full(m1, 2.0 ** -20)
    base[0] = 0.5
    rp, sid, con, ncpv = single_hit_matrix(counts, base, seed=m1)
    smps = []
    for p in pos:
        theta = base.copy()
        theta[p] = 2.0 ** -23   # every row's product stays a power of two
        smps.append(Sample(rp, sid, con, ncpv, theta, 4.0, largest=p))
    assert all(s.m1 == m1 for s in smps)
    warps, lanes = {(p % THREADS) // 32 for p in pos}, {p % 32 for p in pos}
    if m1 >= THREADS:
        assert warps == set(range(THREADS // 32))
    if m1 > 32:
        assert {0, 31} <= lanes
    return smps


@functools.lru_cache(maxsize=None)
def threshold_sample():
    """threshold_matrix with its two hitless transcripts (theta_old = 1e-7 and the double below) named by zero-conprb
    hits in row 0, which leave every row sum unchanged"""
    rp, sid, con, ncpv, theta, M, n0, picks = threshold_matrix()
    hitless = [t for t in range(1, M + 1) if t not in set(np.abs(sid))]
    assert [theta[t] for t in hitless] == [1e-7, float(np.nextafter(1e-7, 0.0))]
    k = len(hitless)
    rp = np.r_[rp[:1], rp[1:] + k].astype(np.uint64)
    sid = np.r_[sid[:1], hitless, sid[1:]].astype(np.int32)
    con = np.r_[con[:1], np.zeros(k), con[1:]]
    return Sample(rp, sid, con, ncpv, theta, n0, picks=picks, M=M)


# ------------------------------------------------------------------------------------------------------------------
# 4. many samples in one launch
# ------------------------------------------------------------------------------------------------------------------
DEG_OF_G = {1: 2, 2: 5, 4: 11, 8: 23, 16: 47, 32: 60}   # a constant degree d with lanes_per_row = G (mean d + 1)


@functools.lru_cache(maxsize=None)
def many_case(sms):
    """2 sms + 1 samples of every G with 1 to 3 tiles, m1 between a few and 3000 in no relation to their size"""
    rng = np.random.default_rng(sms)
    smps = []
    for i in range(2 * sms + 1):
        G = (1, 2, 4, 8, 16, 32)[i % 6]
        d = DEG_OF_G[G]
        k = int(rng.integers(1, 4))
        per_tile = min(ROW_CAP, HIT_CAP // d)
        N = per_tile * (k - 1) + int(rng.integers(1, per_tile + 1))
        smp = from_exact(exact_matrix(np.full(N, d), seed=500 + i, Mr=int(rng.integers(2 * d, 3000))))
        assert smp.G == G and len(smp.tiles) == k
        smps.append(smp)
    assert {s.G for s in smps} == {1, 2, 4, 8, 16, 32} and {len(s.tiles) for s in smps} == {1, 2, 3}
    return smps


def claim_order(smps, live):
    """batch_run's launch order: largest H + N first, stable"""
    return sorted(live, key=lambda s: -(smps[s].H + smps[s].N))


# ------------------------------------------------------------------------------------------------------------------
# 5. fixed-point matrices: every round exactly (2^m, 0, 0)
# ------------------------------------------------------------------------------------------------------------------
def fixed_point_matrix(fams, seed, perturb=None, unnamed=9):
    """fams [(k, j)]: a family of d = 2^k transcripts and d 2^j rows, each row naming all d with equal products and
    ncpv = 0, so each transcript of the family gets count 2^j.  n0 is the power of two that takes the total to 2^m,
    theta = count / 2^m, and the matrix is a fixed point: theta unchanged, stats (2^m, 0, 0).  `perturb` doubles the
    theta of that family: its products stay equal within a row, so round 1 lands on the fixed point with bChange 0.5
    and totNum = d.  `unnamed` transcripts without hits have theta 0."""
    rng = np.random.default_rng(seed)
    R = sum(2 ** (k + j) for k, j in fams)
    n0 = next(2 ** e for e in range(60) if (R + 2 ** e) & (R + 2 ** e - 1) == 0)
    m = (R + n0).bit_length() - 1
    named = sum(2 ** k for k, _ in fams)
    M = named + unnamed
    ids = rng.permutation(M)[:named] + 1
    theta = np.zeros(M + 1)
    theta[0] = n0 / 2.0 ** m
    rows = []
    o = 0
    for f, (k, j) in enumerate(fams):
        d = 2 ** k
        fam = ids[o:o + d]
        o += d
        theta[fam] = 2.0 ** (j - m) * (2.0 if f == perturb else 1.0)
        for _ in range(d * 2 ** j):
            q = int(rng.integers(3, 40))
            rows.append((rng.permutation(fam), 2.0 ** (j - q) / theta[fam]))   # products 2^(j - q) each
    order = rng.permutation(len(rows))
    degs = [len(rows[r][0]) for r in order]
    sid = np.concatenate([rows[r][0] for r in order]) * np.where(rng.random(sum(degs)) < 0.5, 1, -1)
    conprb = np.concatenate([rows[r][1] for r in order])
    row_ptr = np.r_[0, np.cumsum(degs)].astype(np.uint64)
    assert theta.min() == 0 and theta[theta > 0].min() >= 1e-7
    return Sample(row_ptr, sid, conprb, np.zeros(len(degs)), theta, float(n0), total=2.0 ** m,
                  d_perturbed=2 ** fams[perturb][0] if perturb is not None else 0)


FP_FAMILIES = {   # by tile count (fp_case checks it)
    1: [(5, 0), (4, 1)],             # 64 rows, 1536 hits, n0 = 64: G = 16
    2: [(0, 8), (1, 7), (2, 6)],     # 768 rows, 1792 hits, n0 = 256: G = 2
    3: [(3, 6), (2, 6)],             # 768 rows, 5120 hits, n0 = 256: G = 4
}


@functools.lru_cache(maxsize=None)
def fp_case(n_tiles, perturbed):
    fams = FP_FAMILIES[n_tiles]
    smp = fixed_point_matrix(fams, seed=60 + n_tiles, perturb=len(fams) - 1 if perturbed else None)
    assert len(smp.tiles) == n_tiles
    return smp


def converged_sample():
    rp, sid, con, ncpv, theta, M, n0 = converged_matrix()
    return Sample(rp, sid, con, ncpv, theta, n0, total=64.0, d_perturbed=0)


def stop_slots(k):
    """(sample, min_round, max_round, launch in which it stops, rounds it runs) for k rounds per launch"""
    out = []
    fixed = [fp_case(t, False) for t in (1, 2, 3)]
    pert = [fp_case(t, True) for t in (1, 2, 3)]
    mins = [(FIRST + 2 * k - 1, 1), (FIRST + 2 * k, 2)]           # a launch's last round, the next launch's first
    if k >= 3:
        mins.append((FIRST + k + k // 2, 1))                       # inside a launch
    for i, (mn, launch) in enumerate(mins):
        out.append((fixed[i % 3], mn, 10000, launch, mn - FIRST + 1))
    out.append((converged_sample(), FIRST + 2 * k - 1, 10000, 1, 2 * k))
    for i, smp in enumerate(pert):
        out.append((smp, 1, FIRST, 0, 1))                          # max_round = first round: stops with totNum > 0
        out.append((smp, 5, 10000, 0 if k >= 2 else 1, 2))         # min_round below the first round
    out.append((fixed[k % 3], 5, 10000, 0, 1))
    return out


# ------------------------------------------------------------------------------------------------------------------
# 6. sum < 1e-300
# ------------------------------------------------------------------------------------------------------------------
def all_clamped_sample():
    x = exact_matrix(np.zeros(0, np.int64), seed=1, clamp=[("all", d) for d in (1, 2, 3, 5, 9, 40)] * 50, n0=0)
    return from_exact(x)


# ------------------------------------------------------------------------------------------------------------------
# every sample, for the CPU checks
# ------------------------------------------------------------------------------------------------------------------
def exact_samples():
    out = [(f"lane-{T}-{'above' if a else 'at'}", lane_case(T, a)) for T, a in LANE_CASES]
    out += [(f"tile-{n}", tile_case(n)) for n in TILE_CASES]
    out += [(f"mstep-{m1}-{s.largest}", s) for m1 in M1_CASES for s in mstep_case(m1)]
    out += [("threshold", threshold_sample())]
    out += [(f"fp-{t}-{p}", fp_case(t, p)) for t in (1, 2, 3) for p in (False, True)]
    out += [("converged", converged_sample())]
    return out


def _row_sums(smp):
    """per row: (terms of at least 2^-200, exact sum of the terms below 2^-200 that survive the clamp)"""
    row_ptr, sid, conprb, ncpv = smp.m
    rp = row_ptr.astype(np.int64)
    prod = smp.theta[np.abs(sid)] * conprb
    prod[prod < EPS] = 0.0
    f0 = smp.theta[0] * ncpv
    f0[f0 < EPS] = 0.0
    for i in range(smp.N):
        terms = [Fraction(float(v)) for v in prod[rp[i]:rp[i + 1]] if v] + ([Fraction(float(f0[i]))] if f0[i] else [])
        tiny = sum((v for v in terms if v < Fraction(2) ** -200), Fraction(0))
        yield i, sum(terms, Fraction(0)) - tiny, tiny


def _pow2(f):
    return f > 0 and (f.numerator & (f.numerator - 1)) == 0 and (f.denominator & (f.denominator - 1)) == 0


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
def test_builders_are_compact():
    smps = [s for _, s in exact_samples()] + many_case(NOMINAL_SMS) + [lone_epsilon_sample(), all_clamped_sample()]
    for smp in smps:
        named = np.zeros(len(smp.theta), bool)
        named[np.abs(smp.m[1])] = True
        assert not smp.theta[1:][~named[1:]].any()
        assert smp.m1 <= THETA_CAP and smp.H <= 1 << 20 and len(smp.tiles) >= 1


@pytest.mark.parametrize("name", [n for n, _ in exact_samples() if not n.startswith("mstep")] + ["many", "mstep"])
def test_row_sums_are_powers_of_two(name):
    if name == "many":
        smps = many_case(NOMINAL_SMS)
    elif name == "mstep":
        smps = [s for n, s in exact_samples() if n.startswith("mstep")]
    else:
        smps = [dict(exact_samples())[name]]
    for smp in smps:
        kept = 0
        for i, big, tiny in _row_sums(smp):
            if big == 0:   # only the all-clamped rows of exact_matrix
                assert tiny == 0 and smp.clamp[i - smp.n_regular][0] == "all"
                continue
            assert _pow2(big), f"row {i}"
            if tiny:       # exact_matrix's kept clamp edge: far below half an ulp of the sum
                assert tiny == Fraction(EPS) and tiny * 2 ** 60 < big
                kept += 1
        assert kept == sum(s[0] in ("keep", "noise_keep") for s in getattr(smp, "clamp", ()))


def test_lone_epsilon_row():
    """the one row of the sample that is no power of two sums to exactly 1e-300; K12's weight is 1 - 2^-53 there"""
    smp = lone_epsilon_sample()
    sums = list(_row_sums(smp))
    assert all(_pow2(big) and tiny == 0 for _, big, tiny in sums[:-1])
    assert sums[-1][1:] == (Fraction(0), Fraction(EPS))
    assert LONE in (1.0, 1.0 - 2.0 ** -53)


@pytest.mark.parametrize("name", [n for n, _ in exact_samples() if not n.startswith("mstep-12288")])
def test_oracle_does_not_depend_on_its_order(oracle, name):
    smp = dict(exact_samples())[name]
    c1, p1, q1 = oracle.estep(*smp.m, smp.theta, want_post=True, n_threads=1)
    c16, p16, q16 = oracle.estep(*smp.m, smp.theta, want_post=True, n_threads=16)
    _eq(c1, c16)
    _eq(p1, p16)
    _eq(q1, q16)
    for t, want in getattr(smp, "edges", ()):
        assert c1[t] == want


@pytest.mark.parametrize("n_tiles", [1, 2, 3])
@pytest.mark.parametrize("perturbed", [False, True])
def test_fixed_point_matrices(oracle, n_tiles, perturbed):
    """70 oracle rounds: theta stays the fixed point and every round is (2^m, 0, 0), after a perturbed first round of
    (2^m, 0.5, d)"""
    smp = fp_case(n_tiles, perturbed)
    theta, stats, stopped = oracle.em_rounds(*smp.m, smp.theta, smp.n0, FIRST, 70, 1000, 10000)
    assert not stopped and len(stats) == 70
    want = [(smp.total, 0.0, 0)] * 70
    if perturbed:
        want[0] = (smp.total, 0.5, smp.d_perturbed)
        _eq(theta, fp_case(n_tiles, False).theta)
    else:
        _eq(theta, smp.theta)
    assert stats == want


def test_converged_matrix_is_a_fixed_point(oracle):
    smp = converged_sample()
    theta, stats, _ = oracle.em_rounds(*smp.m, smp.theta, smp.n0, FIRST, 70, 1000, 10000)
    _eq(theta, smp.theta)
    assert stats == [(64.0, 0.0, 0)] * 70


def test_cases_reach_their_edges():
    """the builders assert their own edges; across the cases: G = 1..32, tiles closed by rows and by hits, 1, 2 and 3
    tiles, the fixed points' G and tile counts, the claim order of the many-sample launch"""
    assert {lane_case(T, a).G for T, a in LANE_CASES} == {1, 2, 4, 8, 16, 32}
    assert [len(tile_case(n).tiles) for n in ("one", "hits", "rows")] == [1, 2, 3]
    assert [fp_case(t, False).G for t in (1, 2, 3)] == [16, 2, 4] and converged_sample().G == 1
    smps = many_case(NOMINAL_SMS)
    live = [s for s in range(len(smps)) if s != len(smps) // 2]
    m1 = [smps[s].m1 for s in claim_order(smps, live)]
    assert any(a < b for a, b in zip(m1, m1[1:])) and any(a > b for a, b in zip(m1, m1[1:]))
    odd = [len(smps[s].tiles) % 2 for s in claim_order(smps, live)]
    assert 0 < sum(odd) < len(odd)
    for k in (1, 2, 3, CHUNK):
        slots = stop_slots(k)
        assert {len(s.tiles) for s, *_ in slots} == {1, 2, 3}


def test_threshold_sample(oracle):
    """the threshold transcripts land where they claim in the oracle's M-step, with the zero-conprb hits in place"""
    smp = threshold_sample()
    counts = oracle.estep(*smp.m, smp.theta)
    th, (s, b, tot) = oracle.mstep(counts, smp.theta, smp.n0)
    assert s == 2.0 ** 14
    ch = _change(th, smp.theta)
    assert ch[1] == 0.001 and ch[2] < 0.001 and ch[3] == 0.001 and ch[4] < 0.001
    assert smp.theta[5] == 1e-7 and smp.theta[6] < 1e-7 and counts[5] == counts[6] == 0
    assert tot == 2 + 1 + int(ch[0] >= 0.001) + int(ch[smp.M] >= 0.001)


def test_mstep_largest_change(oracle):
    for m1 in M1_CASES:
        for smp in mstep_case(m1):
            th, st = oracle.mstep(oracle.estep(*smp.m, smp.theta), smp.theta, smp.n0)
            changes = np.where(smp.theta >= 1e-7, _change(th, smp.theta), 0.0)
            assert int(np.argmax(changes)) == smp.largest and st[1] == changes[smp.largest]


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sm_count(built):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def round1_exact(ctx, oracle, smps, remove=None):
    """every sample's first round in one launch: stats and theta == oracle.estep + oracle.mstep"""
    import rsem_b200
    with rsem_b200.Batch(ctx) as b:
        slots = [s.add(b) for s in smps]
        if remove is not None:
            b.remove(slots[remove])
        res = b.run(1)
        assert sorted(res) == sorted(s for i, s in enumerate(slots) if i != remove)
        for i, (slot, smp) in enumerate(zip(slots, smps)):
            if i == remove:
                continue
            th_ref, st_ref = oracle.mstep(oracle.estep(*smp.m, smp.theta), smp.theta, smp.n0)
            assert res[slot] == ([st_ref], False), f"sample {i}"
            _eq(b.final(slot)[0], th_ref)


def final_exact(ctx, oracle, smp, lone=None):
    """the final pass on a fresh slot: theta unchanged, counts (count[0] without n0), post and post0 == oracle.estep"""
    import rsem_b200
    c_ref, p_ref, q_ref = oracle.estep(*smp.m, smp.theta, want_post=True)
    with rsem_b200.Batch(ctx) as b:
        theta, counts, post, post0 = b.final(smp.add(b), posteriors=True)
    if lone is not None:   # oracle: 1e-300 / 1e-300 = 1
        t, j = lone
        assert c_ref[t] == p_ref[j] == 1.0
        assert counts[t] == post[j] == LONE and counts[t] in (1.0, 1.0 - 2.0 ** -53)
        c_ref[t], p_ref[j] = LONE, LONE
    _eq(theta, smp.theta)
    _eq(counts, c_ref)
    _eq(post, p_ref)
    _eq(post0, q_ref)


@gpu
@pytest.mark.parametrize("T,above", LANE_CASES, ids=[f"{T}-{'above' if a else 'at'}" for T, a in LANE_CASES])
def test_lane_groups_exact(ctx, oracle, T, above):
    smp = lane_case(T, above)
    round1_exact(ctx, oracle, [smp])
    final_exact(ctx, oracle, smp)


@gpu
def test_lone_epsilon_row_final(ctx, oracle):
    """the only case on the `sum >= 1e-300` edge: weight 1 - 2^-53 (never 0), every other count and posterior =="""
    smp = lone_epsilon_sample()
    final_exact(ctx, oracle, smp, lone=(smp.lone, smp.lone_hit))


@gpu
@pytest.mark.parametrize("name", TILE_CASES)
def test_tiles_exact(ctx, oracle, name):
    smp = tile_case(name)
    round1_exact(ctx, oracle, [smp])
    final_exact(ctx, oracle, smp)


@gpu
@pytest.mark.parametrize("m1", M1_CASES)
def test_mstep_largest_change_exact(ctx, oracle, m1):
    """the largest change in each warp of the strided loop, at lanes 0 and 31 and at m1 - 1, all in one launch"""
    round1_exact(ctx, oracle, mstep_case(m1))


@gpu
def test_mstep_thresholds_exact(ctx, oracle):
    """changes of exactly 0.001 and one ulp of theta_old away on both sides of theta_new; theta_old = 1e-7 and the
    double below it"""
    smp = threshold_sample()
    round1_exact(ctx, oracle, [smp])
    final_exact(ctx, oracle, smp)


@gpu
def test_many_samples_one_launch_exact(ctx, oracle, sm_count):
    """2 SMs + 1 samples, so CTAs claim several with ring phases that differ from sample to sample; one slot removed
    in the middle"""
    smps = many_case(sm_count)
    round1_exact(ctx, oracle, smps, remove=len(smps) // 2)


@gpu
@pytest.mark.parametrize("k", [1, 2, 3, CHUNK])
def test_rounds_ring_and_stop_rule_exact(ctx, oracle, k):
    """fixed-point and perturbed matrices from round 11 with k rounds per launch: min_round inside a launch, at its
    last round and at the next launch's first; max_round = the first round; min_round below it.  Every round's stats,
    the stop launch, theta, counts and posteriors ==; a stopped sample's later run gives no round and keeps theta"""
    import rsem_b200
    cases = stop_slots(k)
    with rsem_b200.Batch(ctx) as b:
        slots = [smp.add(b, FIRST, mn, mx) for smp, mn, mx, _, _ in cases]
        res = _run_to_end(b, slots, k)
        again = b.run(k)
        for slot, (smp, mn, mx, launch, n_rounds) in zip(slots, cases):
            th_ref, st_ref, stopped = oracle.em_rounds(*smp.m, smp.theta, smp.n0, FIRST, 1000, mn, mx)
            assert stopped and len(st_ref) == n_rounds
            stats, when = res[slot]
            assert stats == st_ref, f"slot {slot}: min_round {mn}, max_round {mx}"
            assert when == launch
            assert again[slot] == ([], True)
            theta, counts, post, post0 = b.final(slot, posteriors=True)
            _eq(theta, th_ref)
            c_ref, p_ref, q_ref = oracle.estep(*smp.m, th_ref, want_post=True)
            _eq(counts, c_ref)
            _eq(post, p_ref)
            _eq(post0, q_ref)
        assert all(v == ([], True) for v in b.run(k).values())


@gpu
def test_sum_below_epsilon_raises_then_an_exact_sample_runs(ctx, oracle):
    import rsem_b200
    bad = all_clamped_sample()
    good = lane_case(12, 0)
    with rsem_b200.Batch(ctx) as b:
        s_bad = bad.add(b)
        with pytest.raises(rsem_b200.RsemB200Error, match=r"EM\.cpp:397"):
            b.run(3)
        b.remove(s_bad)
        s = good.add(b)
        th_ref, st_ref = oracle.mstep(oracle.estep(*good.m, good.theta), good.theta, good.n0)
        assert b.run(1)[s] == ([st_ref], False)
        _eq(b.final(s)[0], th_ref)
