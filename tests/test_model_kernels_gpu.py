"""K1 (conprb_kernel: getConPrb / getNoiseConPrb) and K3 (update_q_kernel, update_kernel, update_coop_kernel:
update / updateNoise) against the CPU oracle, through the C ABI.

The inputs are built here from a seed so that every kernel path runs: transcripts assembled from exons shared by the
isoforms of a gene (reads inside shared exons see the same bases on every hit and take the cooperative path) and from
repeat elements shared across genes (the mean degree that picks 4, 8, 16 or 32 lanes per read), isoforms one
substitution away from a sibling, N bases, poly(A) tails, seed masks, transcripts shorter than the RSPD bin count,
reads of 1-150 bases (and >= 1004 for the unstaged profile), paired mates of different lengths, qualities up to 41 and
up to 93, low-quality reads, reads without hits, and conprb values under the 1e-300 cutoff.

Tolerances:
  * K1 per-hit path: bit-identical to the oracle (the same IEEE operations in the same order).
  * K1 cooperative path: 1e-12 relative (a product of up to a few hundred factors associated as a tree).
  * K3 on dyadic posteriors: every profile / noise / fragment-length cell is a sum of exactly representable terms, so
    bit-identical whatever the order of the atomics; RSPD cells (non-dyadic terms) 1e-12 relative.
  * K3 after K1: 1e-10 relative on every cell, zero cells zero on both sides.
"""
import functools

import numpy as np
import pytest

import ref_model as rm
from rsem_b200.capi import ModelStats

EPS = 1e-300
COMP = np.array([3, 2, 1, 0, 4], np.uint8)
LENS = np.array([1, 2, 3, 4, 5, 6, 7, 8, 9, 15, 16, 17, 63, 64, 65, 100, 150])
LENS_P = np.array([.012] * 9 + [.04] * 3 + [.06] * 3 + [.3, .292])
LONG_LENS = np.array([1004, 1100, 1200])
B_RSPD = 20

# model type, lanes per read the mean degree selects, reads, single-end mate-length distribution, RSPD, P(forward),
# largest quality, reads >= 1004 bases
SPECS = {
    "se_noq_g4": dict(mt=0, G=4, N=150_000, mld=False, rspd=True, ori0=0.6),
    "se_noq_g8": dict(mt=0, G=8, N=20_000, mld=True, rspd=True, ori0=0.05),
    "se_noq_g16": dict(mt=0, G=16, N=12_000, mld=False, rspd=False, ori0=0.5),
    "se_noq_g32": dict(mt=0, G=32, N=8_000, mld=True, rspd=True, ori0=0.7),
    "se_noq_long": dict(mt=0, G=4, N=3_000, mld=False, rspd=True, ori0=0.5, long=True),
    "se_q_g4": dict(mt=1, G=4, N=150_000, mld=True, rspd=True, ori0=0.5, qmax=41),
    "se_q_g8": dict(mt=1, G=8, N=20_000, mld=False, rspd=True, ori0=0.05, qmax=93),
    "se_q_g16": dict(mt=1, G=16, N=12_000, mld=True, rspd=False, ori0=0.5, qmax=41),
    "se_q_g32": dict(mt=1, G=32, N=8_000, mld=False, rspd=True, ori0=0.9, qmax=93),
    "pe_noq_g4": dict(mt=2, G=4, N=150_000, rspd=True, ori0=0.5),
    "pe_noq_g8": dict(mt=2, G=8, N=20_000, rspd=False, ori0=0.5),
    "pe_noq_g16": dict(mt=2, G=16, N=12_000, rspd=True, ori0=0.05),
    "pe_noq_g32": dict(mt=2, G=32, N=8_000, rspd=True, ori0=0.5),
    "pe_q_g4": dict(mt=3, G=4, N=150_000, rspd=True, ori0=0.5, qmax=93),
    "pe_q_g8": dict(mt=3, G=8, N=20_000, rspd=True, ori0=0.05, qmax=41),
    "pe_q_g16": dict(mt=3, G=16, N=12_000, rspd=False, ori0=0.5, qmax=93),
    "pe_q_g32": dict(mt=3, G=32, N=8_000, rspd=True, ori0=0.5, qmax=41),
}
# repeat elements: (transcripts carrying each one, share of the reads drawn from them) per lane-group size
REPEAT = {4: (0, 0.0), 8: (16, 0.35), 16: (30, 0.55), 32: (48, 0.75)}


def lane_group(row_ptr):
    """lanes per read of K1 / K3 from the mean degree (+1 for the noise entry), as upload_hits chooses them"""
    N = len(row_ptr) - 1
    d = int(row_ptr[-1]) / N + 1.0
    return 4 if d <= 5 else 8 if d <= 11 else 16 if d <= 26 else 32


def window_bases(refs, t, d, p, L):
    """bases of the windows (transcript t, strand d, position p in strand coordinates, length L) in read direction,
    concatenated"""
    L = np.asarray(L, np.int64)
    start = np.repeat(np.cumsum(L) - L, L)
    k = np.arange(int(L.sum()), dtype=np.int64) - start
    t, d, p = np.repeat(t, L), np.repeat(d, L), np.repeat(np.asarray(p, np.int64), L)
    off, tot = refs["seq_off"].astype(np.int64)[t], refs["tot_len"].astype(np.int64)[t]
    b = refs["seq"][np.where(d == 0, off + p + k, off + tot - 1 - p - k)]
    return np.where(d == 0, b, COMP[b])


def mate_windows(inp, hits, mate):
    """(transcript, strand, position, length) of one mate's window for each hit index"""
    s = inp.sid[hits]
    t, d = np.abs(s), (s < 0).astype(np.int64)
    read = inp.read_of_hit[hits]
    L = np.diff(inp.reads["off"][mate].astype(np.int64))[read]
    p = inp.pos[hits].astype(np.int64)
    if mate == 1:
        p = inp.refs["tot_len"].astype(np.int64)[t] - p - inp.insertL[hits]
        d = 1 - d
    return t, d, p, L


def uniform_flags(inp):
    """per read: every hit shows it the bases hit 0 shows it (both mates); reads without hits are not uniform"""
    N = len(inp.row_ptr) - 1
    rp = inp.row_ptr.astype(np.int64)
    same = np.ones(N, bool)
    same[rp[1:] == rp[:-1]] = False
    H = int(rp[-1])
    for lo in range(0, H, 100_000):
        hits = np.arange(lo, min(H, lo + 100_000))
        first = rp[inp.read_of_hit[hits]]
        for mate in range(inp.reads["n_mates"]):
            a, b = mate_windows(inp, hits, mate), mate_windows(inp, first, mate)
            if a[3].sum() == 0:
                continue
            eq = window_bases(inp.refs, *a) == window_bases(inp.refs, *b)
            L = a[3]
            ok = np.ones(len(hits), bool)
            nz = L > 0
            ok[nz] = np.logical_and.reduceat(eq, (np.cumsum(L) - L)[nz])
            same[inp.read_of_hit[hits[~ok]]] = False
    return same


class Inputs:
    pass


def _lendist(rng, lb, ub, zero_frac=0.05):
    span = ub - lb
    pdf = np.zeros(span + 1)
    pdf[1:] = rng.random(span) ** 2 + 1e-3
    pdf[1:][rng.random(span) < zero_frac] = 0.0
    pdf /= pdf.sum()
    return dict(lb=lb, ub=ub, span=span, pdf=pdf, cdf=np.cumsum(pdf))


def random_model(rng, mt, M, spec, pro_len, max_len, mw):
    hasq, paired = mt & 1, mt >= 2
    m = dict(model_type=mt, M=M, ori0=spec["ori0"], est_rspd=spec["rspd"], B=B_RSPD)
    if paired:
        m["gld"], m["mld"] = _lendist(rng, 30, 380), _lendist(rng, 0, max_len)
    elif spec.get("mld"):
        m["gld"], m["mld"] = _lendist(rng, 20, 350), _lendist(rng, 0, max_len)
    else:
        m["gld"], m["mld"] = _lendist(rng, 0, max_len), None
    pdf = np.zeros(B_RSPD + 2)
    if spec["rspd"]:
        pdf[1:B_RSPD + 1] = rng.random(B_RSPD) + 0.05
        pdf[1 + rng.integers(0, B_RSPD)] = 0.0
    else:
        pdf[1:B_RSPD + 1] = 1.0
    pdf /= pdf.sum()
    cdf = np.zeros(B_RSPD + 2)
    cdf[1:B_RSPD + 1] = np.cumsum(pdf[1:B_RSPD + 1])
    m["rspd_pdf"], m["rspd_cdf"] = pdf, cdf
    rows = 100 if hasq else pro_len
    p = 10.0 ** rng.uniform(-4.5, -1.2, size=(rows, 5, 5))
    for r in range(4):
        p[:, r, r] = 1.0 - p[:, r, :4].sum(1) + p[:, r, r]
    p[:, 4, :] = 10.0 ** rng.uniform(-35, -0.6, size=(rows, 5))  # reference N: some entries tiny
    m["profile"], m["pro_len"] = p.ravel(), 0 if hasq else pro_len
    m["noise"] = rng.uniform(0.05, 0.4, size=500 if hasq else 5)
    m["mw"] = mw
    return m


@functools.lru_cache(maxsize=None)
def build(name, seed=0):
    """seeded inputs for SPECS[name]: refs, reads, hits, model, uniform flags (numpy only)"""
    spec = SPECS[name]
    mt, N = spec["mt"], spec["N"]
    hasq, paired, long_reads = bool(mt & 1), mt >= 2, spec.get("long", False)
    rng = np.random.default_rng([seed, sum(map(ord, name))])
    # ---- exons: gene exons, tiny exons (shorter than the RSPD bin count), repeat elements, padding
    exons, tx = [], []          # exon sequences; transcripts as lists of exon ids
    variants = []                # (transcript, exon, offset in exon) of single substitutions

    def exon(n):
        s = rng.integers(0, 4, n).astype(np.uint8)
        if n > 20 and rng.random() < 0.1:
            a = rng.integers(0, n - 12)
            s[a:a + rng.integers(1, 13)] = 4
        exons.append(s)
        return len(exons) - 1

    n_genes = 60 if long_reads else 300
    for _ in range(n_genes):
        ne = int(rng.integers(2, 6))
        ids = [exon(int(rng.integers(1100, 1500)) if long_reads else int(rng.integers(40, 600))) for _ in range(ne)]
        isos = []
        for _ in range(int(rng.integers(2, 7))):
            rest = [e for e in ids[1:] if rng.random() < 0.5]
            isos.append([ids[0]] + rest)
        if rng.random() < 0.3:  # a sibling that differs from isoform 0 by one base of the shared exon
            variants.append((len(tx) + len(isos) + 1, ids[0], int(rng.integers(0, len(exons[ids[0]])))))
            isos.append(list(isos[0]))
        tx += isos
    for _ in range(20):
        e = exon(int(rng.integers(5, B_RSPD)))
        tx += [[e], [e]]
    k_rep, p_rep = REPEAT[spec["G"]]
    rep_ids = []
    for _ in range(8 if k_rep else 0):
        e = exon(int(rng.integers(450, 700)))
        rep_ids.append(e)
        for t in rng.choice(len(tx), size=k_rep, replace=False):
            tx[t].insert(int(rng.integers(0, len(tx[t]) + 1)), e)
    n_pad = 2 ** int(np.ceil(np.log2(len(tx) + 3))) - 1 - len(tx)
    for _ in range(n_pad):
        tx.append([exon(B_RSPD * int(rng.integers(1, 15)))])
    M = len(tx)
    assert (M + 1) & M == 0
    # ---- transcripts
    full_len = np.zeros(M + 1, np.int32)
    tot_len = np.zeros(M + 1, np.int32)
    seqs, occ = [], [[] for _ in exons]
    for t, ids in enumerate(tx, start=1):
        s, at = [], 0
        for e in ids:
            occ[e].append((t, at))
            s.append(exons[e])
            at += len(exons[e])
        s = np.concatenate(s)
        full_len[t] = len(s)
        tail = 125 if (t < M - n_pad and rng.random() < 0.15) else 0
        tot_len[t] = len(s) + tail
        seqs.append(np.concatenate([s, np.zeros(tail, np.uint8)]))
    for t, e, o in variants:
        at = dict(occ[e])[t] + o
        seqs[t - 1][at] = (seqs[t - 1][at] + 1 + rng.integers(0, 3)) % 4 if seqs[t - 1][at] < 4 else 0
    seq_off = np.zeros(M + 1, np.uint64)
    seq_off[2:] = np.cumsum(tot_len[1:M].astype(np.uint64))
    words = (full_len[1:].astype(np.int64) - 1) // 32 + 1
    mask_off = np.zeros(M + 1, np.uint64)
    mask_off[2:] = np.cumsum(words[:-1]).astype(np.uint64)
    mask_words = np.zeros(int(words.sum()), np.uint32)
    for t in range(1, M + 1):  # seed-mask bits on 3 % of the positions
        bits = np.nonzero(rng.random(full_len[t]) < 0.03)[0]
        np.bitwise_or.at(mask_words, mask_off[t].astype(np.int64) + bits // 32, (1 << (bits % 32)).astype(np.uint32))
    refs = dict(M=M, seq_off=seq_off, seq=np.concatenate(seqs), full_len=full_len, tot_len=tot_len, mask_off=mask_off,
                mask_words=mask_words, has_polyA=True)
    occ_ptr = np.zeros(len(exons) + 1, np.int64)
    occ_ptr[1:] = np.cumsum([len(o) for o in occ])
    occ_t = np.array([t for o in occ for t, _ in o], np.int64)
    occ_at = np.array([a for o in occ for _, a in o], np.int64)
    elen = np.array([len(e) for e in exons], np.int64)

    # ---- reads: an exon, an offset, a strand, lengths
    def draw_len(n):
        L = rng.choice(LENS, size=n, p=LENS_P)
        if long_reads:
            big = rng.random(n) < 0.5
            L[big] = rng.choice(LONG_LENS, size=int(big.sum()))
        return L

    L1 = draw_len(N)
    L2 = draw_len(N) if paired else np.zeros(N, np.int64)
    il = np.maximum(L1, L2) + rng.integers(0, 250, N) if paired else L1.copy()
    need = il
    gene_pool = np.setdiff1d(np.arange(len(exons)), rep_ids)
    gene_pool = gene_pool[np.argsort(elen[gene_pool], kind="stable")]
    lo = np.searchsorted(elen[gene_pool], need)
    assert np.all(lo < len(gene_pool))
    ex = gene_pool[lo + (rng.random(N) * (len(gene_pool) - lo)).astype(np.int64)]
    if rep_ids:
        rep = rng.random(N) < p_rep
        ex[rep] = rng.choice(rep_ids, size=int(rep.sum()))
    o = (rng.random(N) * (elen[ex] - need + 1)).astype(np.int64)
    d = (rng.random(N) >= spec["ori0"]).astype(np.int64)
    # reads whose window ends (in read direction) on a variant's substituted base, lengths not multiples of 8
    tl = []
    for _, e, s in variants:
        for Lt in (9, 15, 17, 63, 65):
            for dd in (0, 1):
                L2t = int(rng.choice(LENS)) if paired else 0
                ilt = max(Lt, L2t) + int(rng.integers(0, 60)) if paired else Lt
                ot = s - Lt + 1 if dd == 0 else (s if not paired else s + Lt - ilt)
                if ot >= 0 and ot + ilt <= elen[e]:
                    tl.append((e, ot, dd, Lt, L2t, ilt))
    # reverse-strand windows reaching base 0 of transcript 1 (sequence offset 0), forward ones ending on the last base
    # of the last transcript (the tail padding)
    for Lt in (9, 17, 64, 100):
        L2t = Lt // 2 if paired else 0
        e0, e1 = tx[0][0], tx[-1][0]
        if Lt <= elen[e0]:
            tl.append((e0, 0, 1, Lt, L2t, Lt))
        if Lt <= elen[e1]:
            tl.append((e1, elen[e1] - Lt, 0, Lt, L2t, Lt))
    if tl:
        tl = np.array(tl, np.int64)
        ex, o, d = np.concatenate([ex, tl[:, 0]]), np.concatenate([o, tl[:, 1]]), np.concatenate([d, tl[:, 2]])
        L1, L2, il = np.concatenate([L1, tl[:, 3]]), np.concatenate([L2, tl[:, 4]]), np.concatenate([il, tl[:, 5]])
    n_main, N = N, len(ex)
    # hits: every occurrence of the exon
    deg = occ_ptr[ex + 1] - occ_ptr[ex]
    read = np.repeat(np.arange(N), deg)
    k = np.arange(int(deg.sum())) - np.repeat(np.cumsum(deg) - deg, deg)
    ht = occ_t[occ_ptr[ex][read] + k]
    f = occ_at[occ_ptr[ex][read] + k] + o[read]   # forward start of the read / fragment in the transcript
    hd = d[read]
    hp = np.where(hd == 0, f, tot_len[ht].astype(np.int64) - f - il[read])
    # a quarter of the reads get 1-2 hits at random places on random transcripts (either strand, poly(A) included)
    n_ex = np.where((np.arange(N) < n_main) & (rng.random(N) < 0.25), rng.integers(1, 3, N), 0)
    xr = np.repeat(np.arange(N), n_ex)
    t_sorted = np.argsort(tot_len[1:], kind="stable") + 1
    lo = np.searchsorted(tot_len[t_sorted], il[xr])
    xt = t_sorted[lo + (rng.random(len(xr)) * (M - lo)).astype(np.int64)]
    xp = (rng.random(len(xr)) * (tot_len[xt] - il[xr] + 1)).astype(np.int64)
    xd = rng.integers(0, 2, len(xr))
    read, ht, hd, hp = (np.concatenate([a, b]) for a, b in ((read, xr), (ht, xt), (hd, xd), (hp, xp)))
    order = np.argsort(read, kind="stable")
    read, ht, hd, hp = read[order], ht[order], hd[order], hp[order]
    # a few reads without hits
    keep = ~np.isin(read, np.nonzero(rng.random(n_main) < 0.003)[0])
    read, ht, hd, hp = read[keep], ht[keep], hd[keep], hp[keep]
    row_ptr = np.zeros(N + 1, np.uint64)
    row_ptr[1:] = np.cumsum(np.bincount(read, minlength=N))
    inp = Inputs()
    inp.name, inp.mt, inp.M, inp.hasq, inp.paired, inp.seed_len = name, mt, M, hasq, paired, 1
    inp.refs, inp.row_ptr, inp.read_of_hit = refs, row_ptr, read
    inp.sid = np.where(hd == 0, ht, -ht).astype(np.int32)
    inp.pos = hp.astype(np.int32)
    inp.insertL = il[read].astype(np.int32) if paired else None
    # ---- read bases: the window of the read's source exon (first occurrence), sequencing errors, N, garbage reads
    st = occ_t[occ_ptr[ex]]
    sf = occ_at[occ_ptr[ex]] + o
    sp = np.where(d == 0, sf, tot_len[st].astype(np.int64) - sf - il)
    reads = dict(n_mates=2 if paired else 1, has_qual=hasq, off=[], base=[], qual=[])
    for mate, L in enumerate((L1, L2) if paired else (L1,)):
        p = sp if mate == 0 else tot_len[st].astype(np.int64) - sp - il
        b = window_bases(refs, st, d if mate == 0 else 1 - d, p, L).astype(np.uint8)
        n = len(b)
        err = rng.random(n) < 0.02
        b[err] = rng.integers(0, 4, int(err.sum()))
        b[rng.random(n) < 0.005] = 4
        garbage = np.repeat(rng.random(N) < 0.01, L)
        b[garbage] = rng.integers(0, 4, int(garbage.sum()))
        off = np.zeros(N + 1, np.uint64)
        off[1:] = np.cumsum(L)
        reads["off"].append(off)
        reads["base"].append(b)
        if hasq:
            q = np.where(rng.random(n) < 0.7, rng.integers(max(spec["qmax"] - 10, 0), spec["qmax"] + 1, n),
                         rng.integers(0, spec["qmax"] + 1, n)).astype(np.uint8)
            q[0] = spec["qmax"]
            reads["qual"].append(q)
        else:
            reads["qual"].append(None)
    reads["lowq"] = (rng.random(N) < 0.03).astype(np.uint8)
    inp.reads = reads
    max_len = int(max(L1.max(), L2.max()))
    # ---- model: poly(A) transcripts get mw < 1, a few transcripts mw < 1e-300
    mw = np.ones(M + 1)
    mw[1:] = np.where(tot_len[1:] > full_len[1:], rng.uniform(0.3, 1.0, M), 1.0)
    mw[rng.choice(np.arange(1, M + 1), size=3, replace=False)] = [0.0, 1e-310, 2e-300]
    inp.max_len = max_len
    inp.model = random_model(rng, mt, M, spec, max_len + 3, max_len, mw)
    inp.model2 = random_model(rng, mt, M, spec, max_len + 3, max_len, mw)
    inp.gld_lb, inp.gld_span = 40, 300  # statistics range narrower than the inserts: the histogram guard runs
    inp.uni = uniform_flags(inp)
    return inp


# ---- shared helpers ---------------------------------------------------------------------------------------------------
def upload(ctx, inp):
    ctx.upload_hits(inp.row_ptr, inp.sid, inp.M, inp.pos, inp.insertL)
    r = inp.reads
    if inp.paired:
        ctx.upload_reads(r["off"][0], r["base"][0], r["qual"][0], r["lowq"], r["off"][1], r["base"][1], r["qual"][1])
    else:
        ctx.upload_reads(r["off"][0], r["base"][0], r["qual"][0], r["lowq"])
    upload_refs(ctx, inp.refs)


def upload_refs(ctx, s):
    ctx.upload_refs(s["seq_off"], s["seq"], s["full_len"], s["tot_len"], s["mask_off"], s["mask_words"])


def oracle_conprb(oracle, inp, model, refs=None):
    keep = rm.Keep()
    return oracle.calc_conprb(rm.make_model(model, inp.seed_len, keep), rm.make_reads(inp.reads, keep),
                              rm.make_refs(refs or inp.refs, keep), inp.row_ptr, inp.sid, inp.pos, inp.insertL)


def stats_arrays(inp, model):
    hasq = model["model_type"] & 1
    return dict(profile=np.zeros(2500 if hasq else model["pro_len"] * 25), noise=np.zeros(500 if hasq else 5),
                gld=np.zeros(inp.gld_span + 1), rspd=np.zeros(model["B"] + 2))


def model_stats(inp, arrs):
    st = ModelStats()
    st.profile, st.noise_profile = rm._dp(arrs["profile"]), rm._dp(arrs["noise"])
    st.gld_pdf, st.rspd_pdf = rm._dp(arrs["gld"]), rm._dp(arrs["rspd"])
    st.gld_lb, st.gld_span = inp.gld_lb, inp.gld_span
    return st


def oracle_stats(oracle, inp, model, post, post0):
    keep = rm.Keep()
    arrs = stats_arrays(inp, model)
    oracle.update_stats(rm.make_model(model, inp.seed_len, keep), rm.make_reads(inp.reads, keep),
                        rm.make_refs(inp.refs, keep), inp.row_ptr, inp.sid, inp.pos, inp.insertL, post, post0,
                        model_stats(inp, arrs))
    return arrs


def device_round(ctx, inp, model, n0):
    arrs = stats_arrays(inp, model)
    rs = ctx.em_model_round(n0, model_stats(inp, arrs))
    return arrs, rs


def stat_keys(inp, model):
    return ["profile", "noise"] + (["gld"] if inp.paired else []) + (["rspd"] if model["est_rspd"] else [])


def set_model(ctx, inp, model):
    keep = rm.Keep()
    ctx.set_model(rm.make_model(model, inp.seed_len, keep))


def dyadic_conprb(inp, seed=1):
    """conprb in {0, 1, 2, 4}, ncpv topping every row up to a power of two: with a uniform theta of 1 / (M + 1) (itself
    a power of two) every posterior is a dyadic rational"""
    rng = np.random.default_rng(seed)
    N, H = len(inp.row_ptr) - 1, int(inp.row_ptr[-1])
    c = rng.choice([0.0, 1.0, 2.0, 4.0], size=H, p=[0.1, 0.3, 0.3, 0.3])
    nc = rng.choice([0.0, 1.0, 2.0, 4.0], size=N)
    s = nc + np.bincount(inp.read_of_hit, weights=c, minlength=N)
    pos = s > 0
    nc[pos] += 2.0 ** np.ceil(np.log2(s[pos])) - s[pos]
    theta = np.full(inp.M + 1, 1.0 / (inp.M + 1))
    return c, nc, theta


def coop_compare(dev, ref, w):
    """relative error of the cooperative path; entries whose value sits within 1e-11 of the 1e-300 cutoff (before
    the division by mw) may fall on either side of it and are dropped.  -> (max relative error, dropped)"""
    near = lambda v: np.abs(v * w - EPS) <= 1e-11 * EPS
    zd, zr = dev == 0, ref == 0
    flip = zd != zr
    dropped = flip & ((zd & near(ref)) | (zr & near(dev)))
    assert np.array_equal(flip, dropped), f"zero pattern differs at {np.nonzero(flip & ~dropped)[0][:10]}"
    both = ~zd & ~zr
    rel = np.abs(dev[both] - ref[both]) / ref[both]
    return (float(rel.max()) if rel.size else 0.0), int(dropped.sum())


# ---- CPU: the builder reaches what the GPU tests rely on ------------------------------------------------------------
@pytest.mark.parametrize("name", list(SPECS))
def test_builder_inputs(name):
    inp = build(name)
    spec = SPECS[name]
    rp, tot, full = inp.row_ptr.astype(np.int64), inp.refs["tot_len"].astype(np.int64), inp.refs["full_len"]
    N = len(rp) - 1
    assert N >= spec["N"] and lane_group(inp.row_ptr) == spec["G"]
    t = np.abs(inp.sid).astype(np.int64)
    assert np.all(t >= 1) and np.all(t <= inp.M)
    # every hit inside its transcript (both mates), the reverse strand's floor reached on transcript 1
    floor = tail = False
    for mate in range(inp.reads["n_mates"]):
        tt, dd, pp, LL = mate_windows(inp, np.arange(len(t)), mate)
        assert np.all(pp >= 0) and np.all(pp + LL <= tot[tt])
        floor |= np.any((tt == 1) & (dd == 1) & (pp + LL == tot[1]))
        tail |= np.any((tt == inp.M) & (dd == 0) & (pp + LL == tot[inp.M]))
    assert floor and tail
    # both kinds of reads make up a real share of the set, so both K1 modes run in one launch
    share = inp.uni.mean()
    assert 0.2 < share < 0.9, share
    assert np.any(rp[1:] == rp[:-1]) and 0.01 < inp.reads["lowq"].mean() < 0.05
    lens = np.diff(inp.reads["off"][0].astype(np.int64))
    for L in (1, 7, 8, 9, 15, 16, 17, 63, 64, 65, 100, 150):
        assert np.any(lens == L)
    if spec.get("long"):
        assert lens.max() >= 1004 and inp.model["pro_len"] >= 1004
    if inp.paired:
        assert np.any(lens != np.diff(inp.reads["off"][1].astype(np.int64)))
        il = inp.insertL
        assert np.any(il <= inp.gld_lb) and np.any(il > inp.gld_lb + inp.gld_span)
    if inp.hasq:
        assert max(q.max() for q in inp.reads["qual"]) == spec["qmax"]
    assert np.any(full < B_RSPD) and np.any(tot > full) and np.any(inp.refs["seq"] == 4)
    assert np.any(np.concatenate(inp.reads["base"]) == 4)
    assert np.sum(inp.model["mw"] < EPS) == 2


@pytest.mark.parametrize("name", ["se_noq_g8", "pe_q_g16"])
def test_builder_oracle_properties(name, oracle):
    """dyadic conprb give exactly dyadic oracle posteriors; the synthetic tables push some conprb under 1e-300;
    reads flagged uniform really have the same per-hit sequence factor in the oracle"""
    inp = build(name)
    c, nc, theta = dyadic_conprb(inp)
    _, post, post0 = oracle.estep(inp.row_ptr, inp.sid, c, nc, theta, want_post=True)
    scale = 2.0 ** 12
    for v in (post, post0):
        assert np.array_equal(v * scale, np.round(v * scale))
    conprb, ncpv = oracle_conprb(oracle, inp, inp.model)
    assert np.any(conprb == 0) and np.any(conprb > 0) and np.any(ncpv > 0)
    # some zeros come from the cutoff, not only from masks, length limits or mw: same hits with the cutoff lifted
    m = dict(inp.model, profile=inp.model["profile"] * 0 + 1.0, noise=inp.model["noise"] * 0 + 1.0)
    c1, _ = oracle_conprb(oracle, inp, m)
    assert np.sum((conprb == 0) & (c1 > 0)) > 10


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx(built):
    import rsem_b200
    c = rsem_b200.Context(0)
    yield c
    c.close()


@functools.lru_cache(maxsize=None)
def _oracle_conprb_cached(oracle, name, which):
    inp = build(name)
    return oracle_conprb(oracle, inp, getattr(inp, which))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SPECS))
def test_conprb_per_hit_bit_identical(ctx, oracle, name, monkeypatch):
    """RSEM_B200_NO_COOP=1: every read on the per-hit path, the oracle's operations in the oracle's order"""
    monkeypatch.setenv("RSEM_B200_NO_COOP", "1")
    inp = build(name)
    upload(ctx, inp)
    set_model(ctx, inp, inp.model)
    n = ctx.launch_count()
    ctx.calc_conprb()
    assert ctx.launch_count() - n == 1  # one conprb_kernel launch, no uniform flags, no cooperative launch
    conprb, ncpv = ctx.download_conprb()
    c_ref, n_ref = _oracle_conprb_cached(oracle, name, "model")
    bad = np.nonzero(conprb != c_ref)[0]
    assert bad.size == 0, (f"{bad.size} of {len(conprb)} conprb differ, e.g. hit {bad[0]}: "
                           f"{conprb[bad[0]]!r} vs {c_ref[bad[0]]!r}")
    assert np.array_equal(ncpv, n_ref)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SPECS))
def test_conprb_cooperative_path(ctx, oracle, name, monkeypatch):
    """uniform reads take the cooperative product (mode 1), the others the per-hit one (mode 2) in the same call"""
    monkeypatch.delenv("RSEM_B200_NO_COOP", raising=False)
    inp = build(name)
    upload(ctx, inp)
    set_model(ctx, inp, inp.model)
    n = ctx.launch_count()
    ctx.calc_conprb()
    assert ctx.launch_count() - n == 3  # uniform flags + mode 1 + mode 2
    conprb, ncpv = ctx.download_conprb()
    c_ref, n_ref = _oracle_conprb_cached(oracle, name, "model")
    e1, d1 = coop_compare(conprb, c_ref, inp.model["mw"][np.abs(inp.sid)])
    e2, d2 = coop_compare(ncpv, n_ref, inp.model["mw"][0])
    print(f"\n{name}: cooperative K1 max rel err {max(e1, e2):.3g}, {d1 + d2} values at the cutoff dropped")
    assert e1 <= 1e-12 and e2 <= 1e-12 and d1 + d2 <= 3
    # the non-uniform reads went through the per-hit path: bit-identical
    nu = ~inp.uni[inp.read_of_hit]
    assert np.array_equal(conprb[nu], c_ref[nu])
    assert np.array_equal(ncpv[~inp.uni], n_ref[~inp.uni])
    # a second call reuses the uniform flags
    n = ctx.launch_count()
    ctx.calc_conprb()
    assert ctx.launch_count() - n == 2


def _k3_variants(name):
    v = ["default", "no_coop"]
    return v + ["global"] if SPECS[name]["mt"] & 1 else v


K3_EXACT = [(n, v) for n in SPECS for v in _k3_variants(n)]


def _k3_env(monkeypatch, variant):
    monkeypatch.delenv("RSEM_B200_NO_COOP", raising=False)
    monkeypatch.delenv("RSEM_B200_K3", raising=False)
    if variant == "no_coop":
        monkeypatch.setenv("RSEM_B200_NO_COOP", "1")
    if variant == "global":
        monkeypatch.setenv("RSEM_B200_K3", "global")


@pytest.mark.gpu
@pytest.mark.parametrize("name,variant", K3_EXACT)
def test_update_stats_dyadic_exact(ctx, oracle, name, variant, monkeypatch):
    """dyadic posteriors: profile, noise and fragment-length statistics bit-identical to the oracle's whatever order
    the reductions ran in; RSPD cells within 1e-12"""
    _k3_env(monkeypatch, variant)
    inp = build(name)
    c, nc, theta = dyadic_conprb(inp)
    upload(ctx, inp)
    set_model(ctx, inp, inp.model)
    if variant != "no_coop":
        ctx.calc_conprb()   # computes the uniform flags the cooperative K3 kernel reads
    ctx.upload_conprb(c, nc)
    ctx.set_theta(theta)
    got, _ = device_round(ctx, inp, inp.model, 0.0)
    cd, nd = ctx.download_conprb()
    assert np.array_equal(cd, c) and np.array_equal(nd, nc)  # K1 did not run: conprb_valid after upload_conprb
    _, post, post0 = oracle.estep(inp.row_ptr, inp.sid, c, nc, theta, want_post=True)
    ref = oracle_stats(oracle, inp, inp.model, post, post0)
    for k in ("profile", "noise", "gld") if inp.paired else ("profile", "noise"):
        bad = np.nonzero(got[k] != ref[k])[0]
        assert bad.size == 0, f"{k}: {bad.size} cells differ, e.g. {bad[0]}: {got[k][bad[0]]!r} vs {ref[k][bad[0]]!r}"
    if inp.model["est_rspd"]:
        assert np.any(ref["rspd"] > 0)
        assert np.all(np.abs(got["rspd"] - ref["rspd"]) <= 1e-12 * ref["rspd"])
    assert np.any(ref["noise"] > 0) and np.any(ref["profile"] > 0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SPECS))
def test_model_round_after_k1(ctx, oracle, name, monkeypatch):
    """a model round as rounds 1-10 run it: K1 on the fresh model, E-step, K3, M-step"""
    _k3_env(monkeypatch, "default")
    inp = build(name)
    upload(ctx, inp)
    set_model(ctx, inp, inp.model)
    theta = np.random.default_rng(2).random(inp.M + 1) + 0.05
    theta /= theta.sum()
    ctx.set_theta(theta)
    n0 = 25.0
    got, rs = device_round(ctx, inp, inp.model, n0)
    c_ref, n_ref = _oracle_conprb_cached(oracle, name, "model")
    counts, post, post0 = oracle.estep(inp.row_ptr, inp.sid, c_ref, n_ref, theta, want_post=True)
    ref = oracle_stats(oracle, inp, inp.model, post, post0)
    err = _check_stats(got, ref, stat_keys(inp, inp.model))
    print(f"\n{name}: K3 after K1 max rel err {err:.3g}")
    th_ref, (s, b, t) = oracle.mstep(counts, theta, n0)
    assert abs(rs[0] - s) <= 1e-12 * s and abs(rs[1] - b) <= 1e-6 * b + 1e-12 and abs(rs[2] - t) <= 2
    th = ctx.get_theta()
    assert np.all(np.abs(th - th_ref) <= 1e-10 * th_ref + 1e-300)


def _check_stats(got, ref, keys, rtol=1e-10):
    worst = 0.0
    for k in keys:
        zr, zg = ref[k] == 0, got[k] == 0
        assert np.array_equal(zr, zg), f"{k}: zero cells differ at {np.nonzero(zr != zg)[0][:10]}"
        nz = ~zr
        rel = np.abs(got[k][nz] - ref[k][nz]) / ref[k][nz]
        if rel.size:
            assert rel.max() <= rtol, f"{k}: max rel err {rel.max():.3g} at cell {np.nonzero(nz)[0][rel.argmax()]}"
            worst = max(worst, float(rel.max()))
    return worst


@pytest.mark.gpu
def test_new_model_recomputes_conprb(ctx, oracle, monkeypatch):
    """set_model with new tables invalidates conprb: the next model round runs K1 on them"""
    monkeypatch.setenv("RSEM_B200_NO_COOP", "1")
    inp = build("pe_q_g8")
    upload(ctx, inp)
    set_model(ctx, inp, inp.model)
    ctx.calc_conprb()
    set_model(ctx, inp, inp.model2)
    ctx.set_theta(np.full(inp.M + 1, 1.0 / (inp.M + 1)))
    n = ctx.launch_count()
    device_round(ctx, inp, inp.model2, 0.0)
    assert ctx.launch_count() - n >= 3  # K1, E-step, K3, fold, theta update
    conprb, ncpv = ctx.download_conprb()
    c_ref, n_ref = _oracle_conprb_cached(oracle, "pe_q_g8", "model2")
    assert np.array_equal(conprb, c_ref) and np.array_equal(ncpv, n_ref)
    assert not np.array_equal(c_ref, _oracle_conprb_cached(oracle, "pe_q_g8", "model")[0])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["se_q_g4", "pe_noq_g16"])
def test_new_refs_recompute_uniform_flags(ctx, oracle, name, monkeypatch):
    """upload_refs with one substitution in a shared exon: reads that were uniform and are no longer take the
    per-hit path on the next K1 call"""
    monkeypatch.delenv("RSEM_B200_NO_COOP", raising=False)
    inp = build(name)
    upload(ctx, inp)
    set_model(ctx, inp, inp.model)
    ctx.calc_conprb()
    # a uniform read with several hits: change one base in the middle of its window on its last hit
    rp = inp.row_ptr.astype(np.int64)
    cand = np.nonzero(inp.uni & (np.diff(rp) >= 2) & (np.diff(inp.reads["off"][0].astype(np.int64)) >= 60)
                      & (inp.reads["lowq"] == 0))[0]
    i = int(cand[len(cand) // 2])
    j = rp[i + 1] - 1
    t, d, p, L = (int(x[0]) for x in mate_windows(inp, np.array([j]), 0))
    fwd = p + L // 2 if d == 0 else int(inp.refs["tot_len"][t]) - 1 - p - L // 2
    refs2 = dict(inp.refs, seq=inp.refs["seq"].copy())
    at = int(inp.refs["seq_off"][t]) + fwd
    refs2["seq"][at] = (refs2["seq"][at] + 1) % 4
    inp2 = Inputs()
    inp2.__dict__.update(inp.__dict__)
    inp2.refs = refs2
    uni2 = uniform_flags(inp2)
    lost = inp.uni & ~uni2
    assert lost[i] and not np.any(uni2 & ~inp.uni)
    upload_refs(ctx, refs2)
    n = ctx.launch_count()
    ctx.calc_conprb()
    assert ctx.launch_count() - n == 3  # the uniform flags were recomputed
    conprb, ncpv = ctx.download_conprb()
    c_ref, n_ref = oracle_conprb(oracle, inp, inp.model, refs2)
    h = lost[inp.read_of_hit]
    assert np.array_equal(conprb[h], c_ref[h]) and np.array_equal(ncpv[lost], n_ref[lost])
    e, _ = coop_compare(conprb, c_ref, inp.model["mw"][np.abs(inp.sid)])
    assert e <= 1e-12
    upload_refs(ctx, inp.refs)


# ---- the golden data sets with the reference's round-20 model --------------------------------------------------------
@pytest.fixture(scope="module")
def golden(tmp_path_factory, built):
    import golden_util as gu
    import rsem_files as rf
    out = {}
    for name in gu.CASES:
        case = gu.Case(name, tmp_path_factory.mktemp("golden_k13"))
        inp = Inputs()
        inp.name, inp.mt, inp.M, inp.hasq, inp.paired = name, case.rt, case.M, case.hasq, case.paired
        inp.seed_len = case.mp["seedLen"]
        inp.refs, inp.row_ptr, inp.sid, inp.pos, inp.insertL = case.refs, case.row_ptr, case.sid, case.pos, case.insertL
        if not inp.paired:
            inp.insertL = None
        inp.reads = case.reads
        inp.read_of_hit = np.repeat(np.arange(len(case.row_ptr) - 1), np.diff(case.row_ptr.astype(np.int64)))
        inp.gld_lb, inp.gld_span = case.mp["minL"] - 1, case.mp["maxL"] - (case.mp["minL"] - 1)
        inp.model = rf.read_model(case.out("model20"), case.M)
        inp.theta0 = case.theta0()
        out[name] = inp
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["se_noq", "se_q_rspd", "pe_noq", "pe_q_rspd", "se_q_polyA"])
def test_golden_cases(ctx, oracle, golden, name, monkeypatch):
    inp = golden[name]
    c_ref, n_ref = oracle_conprb(oracle, inp, inp.model)
    monkeypatch.setenv("RSEM_B200_NO_COOP", "1")
    upload(ctx, inp)
    set_model(ctx, inp, inp.model)
    ctx.calc_conprb()
    conprb, ncpv = ctx.download_conprb()
    assert np.array_equal(conprb, c_ref) and np.array_equal(ncpv, n_ref)
    monkeypatch.delenv("RSEM_B200_NO_COOP")
    set_model(ctx, inp, inp.model)
    ctx.calc_conprb()
    conprb, ncpv = ctx.download_conprb()
    e1, _ = coop_compare(conprb, c_ref, inp.model["mw"][np.abs(inp.sid)])
    e2, _ = coop_compare(ncpv, n_ref, inp.model["mw"][0])
    assert max(e1, e2) <= 1e-12
    set_model(ctx, inp, inp.model)
    ctx.set_theta(inp.theta0)
    got, _ = device_round(ctx, inp, inp.model, 10.0)
    _, post, post0 = oracle.estep(inp.row_ptr, inp.sid, c_ref, n_ref, inp.theta0, want_post=True)
    ref = oracle_stats(oracle, inp, inp.model, post, post0)
    err = _check_stats(got, ref, stat_keys(inp, inp.model))
    print(f"\n{name}: cooperative K1 max rel err {max(e1, e2):.3g}, K3 max rel err {err:.3g}")
