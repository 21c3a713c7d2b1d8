"""ctypes binding of oracle/librsem_oracle.so - TEST INFRASTRUCTURE (the checker, never the product)."""
import ctypes as C
import os

import numpy as np

from rsem_b200.capi import LenDist, Model, ModelStats, RoundStats  # identical layouts (see rsem_oracle.h)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PATH = os.path.join(ROOT, "oracle", "librsem_oracle.so")


class Reads(C.Structure):
    _fields_ = [("n_mates", C.c_int32), ("has_qual", C.c_int32), ("off", C.POINTER(C.c_uint64) * 2),
                ("base", C.POINTER(C.c_uint8) * 2), ("qual", C.POINTER(C.c_uint8) * 2), ("lowq", C.POINTER(C.c_uint8))]


class Refs(C.Structure):
    _fields_ = [("M", C.c_int32), ("seq_off", C.POINTER(C.c_uint64)), ("seq", C.POINTER(C.c_uint8)),
                ("full_len", C.POINTER(C.c_int32)), ("tot_len", C.POINTER(C.c_int32)),
                ("mask_off", C.POINTER(C.c_uint64)), ("mask_words", C.POINTER(C.c_uint32))]


def _p(a, ct):
    return None if a is None else a.ctypes.data_as(C.POINTER(ct))


def c64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class Oracle:
    def __init__(self):
        self.dll = C.CDLL(PATH)
        self.dll.ro_em_rounds.restype = C.c_int32
        self.dll.ro_mt_next.restype = C.c_uint32

    def estep(self, row_ptr, sid, conprb, ncpv, theta, want_post=False, n_threads=1):
        row_ptr = np.ascontiguousarray(row_ptr, np.uint64); sid = np.ascontiguousarray(sid, np.int32)
        conprb, ncpv, theta = c64(conprb), c64(ncpv), c64(theta)
        N, M = len(row_ptr) - 1, len(theta) - 1
        counts = np.zeros(M + 1)
        post = np.zeros(len(sid)) if want_post else None
        post0 = np.zeros(N) if want_post else None
        self.dll.ro_estep(C.c_uint64(N), _p(row_ptr, C.c_uint64), _p(sid, C.c_int32), _p(conprb, C.c_double),
                          _p(ncpv, C.c_double), _p(theta, C.c_double), C.c_int32(M), _p(counts, C.c_double),
                          _p(post, C.c_double), _p(post0, C.c_double), C.c_int32(n_threads))
        return (counts, post, post0) if want_post else counts

    def mstep(self, counts, theta, n0):
        """-> (new theta, (sum, bchange, totnum)); theta is the one the round started from"""
        counts, theta = c64(counts).copy(), c64(theta).copy()
        st = RoundStats()
        self.dll.ro_mstep(C.c_int32(len(theta) - 1), _p(counts, C.c_double), _p(theta, C.c_double), C.c_double(n0),
                          C.byref(st))
        return theta, (st.sum, st.bchange, st.totnum)

    def em_rounds(self, row_ptr, sid, conprb, ncpv, theta, n0, first_round, max_rounds, min_round, max_round, n_threads=1):
        row_ptr = np.ascontiguousarray(row_ptr, np.uint64); sid = np.ascontiguousarray(sid, np.int32)
        conprb, ncpv = c64(conprb), c64(ncpv)
        theta = c64(theta).copy()
        N, M = len(row_ptr) - 1, len(theta) - 1
        stats = (RoundStats * max(max_rounds, 1))()
        stopped = C.c_int32(0)
        ran = self.dll.ro_em_rounds(C.c_uint64(N), _p(row_ptr, C.c_uint64), _p(sid, C.c_int32), _p(conprb, C.c_double),
                                    _p(ncpv, C.c_double), C.c_int32(M), _p(theta, C.c_double), C.c_double(n0),
                                    C.c_int32(first_round), C.c_int32(max_rounds), C.c_int32(min_round),
                                    C.c_int32(max_round), stats, C.byref(stopped), C.c_int32(n_threads))
        return theta, [(stats[i].sum, stats[i].bchange, stats[i].totnum) for i in range(ran)], bool(stopped.value)

    def calc_conprb(self, model, reads, refs, row_ptr, sid, pos, insertL):
        row_ptr = np.ascontiguousarray(row_ptr, np.uint64); sid = np.ascontiguousarray(sid, np.int32)
        pos = np.ascontiguousarray(pos, np.int32)
        insertL = None if insertL is None else np.ascontiguousarray(insertL, np.int32)
        N = len(row_ptr) - 1
        conprb, ncpv = np.zeros(len(sid)), np.zeros(N)
        self.dll.ro_calc_conprb(C.byref(model), C.byref(reads), C.byref(refs), C.c_uint64(N), _p(row_ptr, C.c_uint64),
                                _p(sid, C.c_int32), _p(pos, C.c_int32), _p(insertL, C.c_int32), _p(conprb, C.c_double),
                                _p(ncpv, C.c_double))
        return conprb, ncpv

    def update_stats(self, model, reads, refs, row_ptr, sid, pos, insertL, post, post0, stats):
        row_ptr = np.ascontiguousarray(row_ptr, np.uint64); sid = np.ascontiguousarray(sid, np.int32)
        pos = np.ascontiguousarray(pos, np.int32)
        insertL = None if insertL is None else np.ascontiguousarray(insertL, np.int32)
        post, post0 = c64(post), c64(post0)
        N = len(row_ptr) - 1
        self.dll.ro_update_stats(C.byref(model), C.byref(reads), C.byref(refs), C.c_uint64(N), _p(row_ptr, C.c_uint64),
                                 _p(sid, C.c_int32), _p(pos, C.c_int32), _p(insertL, C.c_int32), _p(post, C.c_double),
                                 _p(post0, C.c_double), C.byref(stats))

    def mt_first(self, seed, n):
        buf = C.create_string_buffer(624 * 4 + 8)
        self.dll.ro_mt_seed(buf, C.c_uint32(seed))
        return [self.dll.ro_mt_next(buf) for _ in range(n)]

    def chain_seeds(self, seed, n):
        out = np.zeros(n, np.uint32)
        self.dll.ro_chain_seeds(C.c_uint32(seed), C.c_int32(n), _p(out, C.c_uint32))
        return out

    def gibbs_chain(self, row_ptr, sid, conprb, M, n0, init_counts, pseudo_counts, totc, eel, mw, gene_start, burnin,
                    gap, n_samples, seed):
        row_ptr = np.ascontiguousarray(row_ptr, np.uint64); sid = np.ascontiguousarray(sid, np.int32)
        conprb = c64(conprb); init_counts = np.ascontiguousarray(init_counts, np.int32)
        pseudo_counts, eel, mw = c64(pseudo_counts), c64(eel), c64(mw)
        gene_start = np.ascontiguousarray(gene_start, np.int32)
        m = len(gene_start) - 1
        cv = np.zeros((n_samples, M + 1), np.int32)
        sums = [np.zeros(M + 1) for _ in range(4)] + [np.zeros(m)]
        self.dll.ro_gibbs_chain(C.c_uint64(len(row_ptr) - 1), _p(row_ptr, C.c_uint64), _p(sid, C.c_int32),
                                _p(conprb, C.c_double), C.c_int32(M), C.c_double(n0), _p(init_counts, C.c_int32),
                                _p(pseudo_counts, C.c_double), C.c_double(totc), _p(eel, C.c_double), _p(mw, C.c_double),
                                C.c_int32(m), _p(gene_start, C.c_int32), C.c_int32(burnin), C.c_int32(gap),
                                C.c_int32(n_samples), C.c_uint32(seed), _p(cv, C.c_int32),
                                *[_p(s, C.c_double) for s in sums])
        return cv, sums

    def polish_theta(self, theta, eel, mw):
        theta = c64(theta).copy()
        self.dll.ro_polish_theta(C.c_int32(len(theta) - 1), _p(theta, C.c_double), _p(c64(eel), C.c_double), _p(c64(mw), C.c_double))
        return theta
