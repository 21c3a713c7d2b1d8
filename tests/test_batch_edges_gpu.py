"""K12 (rsem_b200_batch_*) at the edges of its layout and launch logic, against the CPU oracle on each sample's full-M matrix
with test_em_batch_gpu's tolerances and comparison.

Each case asserts from its CSR that it reaches the edge it is about.  The two rules of batch_kernels.cu that decide this
are restated here: lanes_per_row (G lanes per row from the mean degree H / N + 1) and cut_tiles (tiles of at most 2048 hits
and 512 rows), together with the sizes of the four 16-byte aligned bulk copies issue_tile puts into a Stage.  A case that
stops reaching its edge fails here instead of passing quietly."""
import numpy as np
import pytest

import synth
from test_em_batch_gpu import _compare, _run_to_end, _sample, ctx  # noqa: F401  (ctx: the module's context fixture)

pytestmark = pytest.mark.gpu

HIT_CAP, ROW_CAP = 2048, 512          # kHitCap, kRowCap
MAX_HITS = 1 << 20                    # kMaxHits
# elements of each Stage array: con, ncp, sid, rp
STAGE = dict(con=HIT_CAP + 4, ncp=ROW_CAP + 4, sid=HIT_CAP + 8, rp=ROW_CAP + 8)
G_THRESHOLDS = (3, 6, 12, 24, 48)


# ---- the rules of batch_kernels.cu, restated -------------------------------------------------------------------------------
def lanes_per_row(N, H):
    mean_deg = H / max(N, 1) + 1.0
    for g, t in zip((1, 2, 4, 8, 16), G_THRESHOLDS):
        if mean_deg <= t:
            return g
    return 32


def cut_tiles(row_ptr):
    """(tile_row, tile_hit) bounds: a tile closes before the row that would take it past 512 rows or 2048 hits"""
    rp = [int(x) for x in row_ptr]
    trow, thit, r0 = [0], [0], 0
    for r in range(len(rp) - 1):
        assert rp[r + 1] - rp[r] <= HIT_CAP
        if r - r0 + 1 > ROW_CAP or rp[r + 1] - rp[r0] > HIT_CAP:
            trow.append(r)
            thit.append(rp[r])
            r0 = r
    trow.append(len(rp) - 1)
    thit.append(rp[-1])
    return trow, thit


def copy_elems(rs, re, hs, he):
    """elements each bulk copy of issue_tile moves: from the aligned-down start, rounded up to 16 bytes"""
    def r16(n, size):
        return -(-n * size // 16) * 16 // size
    return dict(sid=r16(he - (hs & ~3), 4), con=r16(he - (hs & ~1), 8), rp=r16(re + 1 - (rs & ~3), 4),
                ncp=r16(re - (rs & ~1), 8))


def tiles(row_ptr):
    """[(rs, re, hs, he, copy sizes)] of a sample; every copy fits its Stage array"""
    trow, thit = cut_tiles(row_ptr)
    out = []
    for k in range(len(trow) - 1):
        c = copy_elems(trow[k], trow[k + 1], thit[k], thit[k + 1])
        assert all(c[a] <= STAGE[a] for a in STAGE), (k, c)
        out.append((trow[k], trow[k + 1], thit[k], thit[k + 1], c))
    return out


# ---- samples ---------------------------------------------------------------------------------------------------------------
def _from_degrees(oracle, deg, M, seed, n0=30.0):
    """a sample whose row k has deg[k] hits on a run of consecutive transcript ids (an isoform family), after oracle round 1"""
    rng = np.random.default_rng(seed)
    deg = np.asarray(deg, np.int64)
    N = len(deg)
    row_ptr = np.zeros(N + 1, np.uint64)
    row_ptr[1:] = np.cumsum(deg)
    H = int(row_ptr[-1])
    start = rng.integers(1, M - deg + 2)
    within = np.arange(H) - np.repeat(row_ptr[:-1].astype(np.int64), deg)
    sid = (np.repeat(start, deg) + within).astype(np.int32)
    sid *= np.where(rng.random(H) < 0.5, 1, -1).astype(np.int32)
    conprb = 10.0 ** rng.uniform(-30, -3, size=H)
    conprb[rng.random(H) < 0.01] = 0.0
    ncpv = 10.0 ** rng.uniform(-40, -8, size=N)
    theta0 = synth.init_theta(M, n0, N + n0)
    theta1 = oracle.em_rounds(row_ptr, sid, conprb, ncpv, theta0, n0, 1, 1, 20, 10000)[0]
    return dict(m=(row_ptr, sid, conprb, ncpv), theta=theta1, n0=n0)


def _degrees_summing_to(N, H, seed):
    """N row degrees >= 1 that sum to exactly H"""
    return 1 + np.random.default_rng(seed).multinomial(H - N, np.full(N, 1.0 / N))


def _G(smp):
    row_ptr = smp["m"][0]
    return lanes_per_row(len(row_ptr) - 1, int(row_ptr[-1]))


# ---- 1. lanes per row ----------------------------------------------------------------------------------------------------
def test_lanes_per_row_thresholds(ctx, oracle):
    """for every threshold t of lanes_per_row, a sample whose mean degree H / N + 1 is exactly t and one just above it, so
    that G = 1, 2, 4, 8, 16 and 32 all run, each with tiles of more rows than one pass of the CTA covers; the rounds and the
    final pass (posteriors)"""
    import rsem_b200
    N, M = 1500, 4000
    smps, want = [], []
    for k, (t, g) in enumerate(zip(G_THRESHOLDS, (1, 2, 4, 8, 16))):
        for extra, gg in ((0, g), (1, 2 * g)):
            H = (t - 1) * N + extra
            smp = _from_degrees(oracle, _degrees_summing_to(N, H, seed=10 * k + extra), M, seed=10 * k + extra)
            assert int(smp["m"][0][-1]) == H and _G(smp) == gg
            # rows per tile exceed the rows one pass of the 16 warps covers (16 * 32 / G), so the row stride is taken
            # (G = 1 covers 512 rows, a whole tile, in one pass)
            if gg > 1:
                assert max(re - rs for rs, re, _, _, _ in tiles(smp["m"][0])) > 16 * 32 // gg
            smps.append(smp)
            want.append(gg)
    assert sorted(set(want)) == [1, 2, 4, 8, 16, 32]
    with rsem_b200.Batch(ctx) as b:
        slots = [b.add(*s["m"], s["theta"], s["n0"], 2, 20, 150) for s in smps]
        res = _run_to_end(b, slots, 16)
        for s, smp in zip(slots, smps):
            _compare(oracle, b, s, smp, 20, 150, res[s][0])


# ---- 2. stage capacity ---------------------------------------------------------------------------------------------------
def _stage_degrees(filler_deg, n_fill):
    """row 0: 3 hits; rows 1 and 2: 2048 hits each, a tile apiece, row 2's starting at hit 2051; rows 3..514: 512 rows of 4
    hits, one tile starting at row 3 and hit 4099; then filler rows that set G"""
    return [3, HIT_CAP, HIT_CAP] + [4] * ROW_CAP + [filler_deg] * n_fill


@pytest.mark.parametrize("filler_deg,n_fill,G", [(1, 6000, 1), (200, 400, 32)])
def test_largest_stage_copies(ctx, oracle, filler_deg, n_fill, G):
    """tiles whose four bulk copies reach their largest sizes: sid 2052 of 2056 ints (2048 hits from hit = 3 mod 4), con 2050
    of 2052 doubles (2048 hits from an odd hit), rp 516 of 520 words (512 rows from row = 3 mod 4), ncp 514 of 516 doubles
    (512 rows from an odd row); rows of exactly 2048 hits"""
    import rsem_b200
    smp = _from_degrees(oracle, _stage_degrees(filler_deg, n_fill), 4000, seed=filler_deg)
    row_ptr = smp["m"][0]
    assert _G(smp) == G
    ts = tiles(row_ptr)
    big_row = [t for t in ts if t[1] - t[0] == 1 and t[3] - t[2] == HIT_CAP]
    assert len(big_row) == 2 and big_row[1][2] % 4 == 3
    assert big_row[1][4]["sid"] == 2052 and big_row[1][4]["con"] == 2050
    rs, re, hs, he, c = next(t for t in ts if t[0] == 3)
    assert (re - rs, hs % 4, he - hs) == (ROW_CAP, 3, HIT_CAP)
    assert c == dict(sid=2052, con=2050, rp=516, ncp=514)
    for a in STAGE:   # no tile of the sample copies more
        assert max(t[4][a] for t in ts) == c[a]
    with rsem_b200.Batch(ctx) as b:
        s = b.add(*smp["m"], smp["theta"], smp["n0"], 2, 20, 150)
        res = _run_to_end(b, [s], 16)
        _compare(oracle, b, s, smp, 20, 150, res[s][0])


# ---- 3. hit cap ----------------------------------------------------------------------------------------------------------
def test_hit_cap(ctx, oracle):
    """a sample of exactly 2^20 hits runs in the batch next to a small one; one more hit is refused at sample_bytes and at
    add with ERR_UNSUPPORTED"""
    import rsem_b200
    from rsem_b200.capi import RSEM_B200_ERR_UNSUPPORTED
    N, M = MAX_HITS // 4, 12000
    big = _from_degrees(oracle, np.full(N, 4), M, seed=20)
    row_ptr, sid, conprb, ncpv = big["m"]
    m = len(np.unique(np.abs(sid)))
    assert int(row_ptr[-1]) == MAX_HITS and m <= 12287
    assert _G(big) == 2 and len(tiles(row_ptr)) == MAX_HITS // HIT_CAP
    small = _sample(oracle, 1000, 60, 3, seed=21)
    over_rp = row_ptr.copy()
    over_rp[-1] += 1
    over = (over_rp, np.append(sid, np.int32(1)), np.append(conprb, 1e-5), ncpv)
    with rsem_b200.Batch(ctx) as b:
        assert b.sample_bytes(row_ptr, m) > 0
        for call in (lambda: b.sample_bytes(over_rp, m), lambda: b.add(*over, big["theta"], big["n0"], 2, 6, 6)):
            with pytest.raises(rsem_b200.RsemB200Error) as e:
                call()
            assert f"error {RSEM_B200_ERR_UNSUPPORTED}:" in str(e.value) and "2^20 hits" in str(e.value)
        s_big = b.add(*big["m"], big["theta"], big["n0"], 2, 6, 6)
        s_small = b.add(*small["m"], small["theta"], small["n0"], 2, 20, 100)
        res = _run_to_end(b, [s_big, s_small], 64)
        assert len(res[s_big][0]) == 5
        _compare(oracle, b, s_big, big, 6, 6, res[s_big][0])
        _compare(oracle, b, s_small, small, 20, 100, res[s_small][0])


# ---- 4. stats with a hole in the slots --------------------------------------------------------------------------------------
def test_run_64_rounds_with_an_empty_middle_slot(ctx, oracle):
    """64 rounds per launch (rsem-run-em-batch's CHUNK) over slots 0..4 with slot 2 removed and left empty; the launch order
    (largest first) is not the slot order, so each sample's stats must be taken from its launch position and put at its
    slot; one sample runs past the first launch"""
    import rsem_b200
    specs = [(600, 40, 3, 20, 40), (1500, 120, 5, 70, 100), (900, 60, 4, 20, 60), (3000, 200, 7, 20, 150),
             (2200, 150, 6, 2, 64)]    # N, M, degree, MIN_ROUND, MAX_ROUND
    smps = [_sample(oracle, N, M, d, seed=40 + k) for k, (N, M, d, _, _) in enumerate(specs)]
    with rsem_b200.Batch(ctx) as b:
        slots = [b.add(*s["m"], s["theta"], s["n0"], 2, lo, hi) for s, (_, _, _, lo, hi) in zip(smps, specs)]
        assert slots == [0, 1, 2, 3, 4]
        b.remove(2)
        live = [0, 1, 3, 4]
        size = {s: int(smps[s]["m"][0][-1]) + len(smps[s]["m"][0]) - 1 for s in live}   # H + N, batch_run's order
        order = sorted(live, key=lambda s: -size[s])
        assert order != live and order.index(1) > 0
        res = _run_to_end(b, live, 64)
        assert 69 <= len(res[1][0]) <= 99 and res[1][1] == 1     # MIN_ROUND 70, MAX_ROUND 100: the second launch
        assert len(res[4][0]) <= 63 and res[4][1] == 0
        for s in live:
            lo, hi = specs[s][3], specs[s][4]
            _compare(oracle, b, s, smps[s], lo, hi, res[s][0])
