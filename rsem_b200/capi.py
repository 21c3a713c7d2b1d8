"""ctypes mirror of include/rsem_b200.h (one Python method per C entry point, same names)."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "librsem_b200.so")


class RsemB200Error(RuntimeError):
    pass


class LenDist(C.Structure):
    _fields_ = [("lb", C.c_int32), ("ub", C.c_int32), ("span", C.c_int32),
                ("pdf", C.POINTER(C.c_double)), ("cdf", C.POINTER(C.c_double))]


class Model(C.Structure):
    _fields_ = [("model_type", C.c_int32), ("M", C.c_int32), ("seed_len", C.c_int32), ("est_rspd", C.c_int32),
                ("rspd_B", C.c_int32), ("has_mld", C.c_int32), ("pro_len", C.c_int32), ("reserved", C.c_int32),
                ("ori", C.c_double * 2), ("gld", LenDist), ("mld", LenDist),
                ("rspd_pdf", C.POINTER(C.c_double)), ("rspd_cdf", C.POINTER(C.c_double)),
                ("profile", C.POINTER(C.c_double)), ("noise_profile", C.POINTER(C.c_double)),
                ("mw", C.POINTER(C.c_double))]


class ModelStats(C.Structure):
    _fields_ = [("profile", C.POINTER(C.c_double)), ("noise_profile", C.POINTER(C.c_double)),
                ("gld_pdf", C.POINTER(C.c_double)), ("gld_lb", C.c_int32), ("gld_span", C.c_int32),
                ("rspd_pdf", C.POINTER(C.c_double))]


class RoundStats(C.Structure):
    _fields_ = [("sum", C.c_double), ("bchange", C.c_double), ("totnum", C.c_int64)]


class GibbsParams(C.Structure):
    _fields_ = [("M", C.c_int32), ("burnin", C.c_int32), ("gap", C.c_int32), ("n_chains", C.c_int32),
                ("chain_samples", C.POINTER(C.c_int32)), ("chain_seeds", C.POINTER(C.c_uint32)),
                ("n0", C.c_double), ("init_counts", C.POINTER(C.c_int32)), ("pseudo_counts", C.POINTER(C.c_double)),
                ("totc", C.c_double), ("eel", C.POINTER(C.c_double)), ("mw", C.POINTER(C.c_double)),
                ("n_genes", C.c_int32), ("gene_start", C.POINTER(C.c_int32))]


class GibbsOut(C.Structure):
    _fields_ = [("count_vectors", C.POINTER(C.c_int32)), ("sum_c", C.POINTER(C.c_double)),
                ("sum_c2", C.POINTER(C.c_double)), ("sum_tpm", C.POINTER(C.c_double)),
                ("sum_fpkm", C.POINTER(C.c_double)), ("sum_gene_c2", C.POINTER(C.c_double))]


class GibbsStats(C.Structure):
    _fields_ = [("device_ms", C.c_double), ("worker_ctas", C.c_int32), ("launches", C.c_int32)]


class GibbsBatchStats(C.Structure):
    _fields_ = [("device_ms", C.c_double), ("worker_ctas", C.c_int32), ("teams", C.c_int32), ("jobs", C.c_int64),
                ("chain_cycles", C.c_uint64), ("sample_cycles", C.c_uint64)]


class SimParams(C.Structure):
    _fields_ = [("model_type", C.c_int32), ("M", C.c_int32), ("seed", C.c_uint32), ("exact_body", C.c_int32),
                ("N", C.c_uint64), ("window_words", C.c_uint64), ("theta_cdf", C.POINTER(C.c_double)),
                ("ori_prob0", C.c_double), ("gld", LenDist), ("mld", LenDist), ("has_mld", C.c_int32),
                ("est_rspd", C.c_int32), ("rspd_off", C.POINTER(C.c_uint64)), ("rspd_cdf", C.POINTER(C.c_double)),
                ("qd_init_cdf", C.POINTER(C.c_double)), ("qd_tran_cdf", C.POINTER(C.c_double)),
                ("pro_rows", C.c_int32), ("reserved", C.c_int32), ("profile_cdf", C.POINTER(C.c_double)),
                ("noise_cdf", C.POINTER(C.c_double)), ("seq_off", C.POINTER(C.c_uint64)),
                ("seq", C.POINTER(C.c_uint8)), ("tot_len", C.POINTER(C.c_int32)), ("full_len", C.POINTER(C.c_int32))]


class SimStats(C.Structure):
    _fields_ = [("generate_ms", C.c_double), ("resolve_ms", C.c_double), ("reads_ms", C.c_double),
                ("copy_ms", C.c_double), ("words", C.c_uint64), ("windows", C.c_uint64)]


class SimDevicesStats(C.Structure):
    _fields_ = [("sum", SimStats), ("jump_ms", C.c_double), ("handoff_ms", C.c_double)]


class CiParams(C.Structure):
    _fields_ = [("M", C.c_int32), ("n_genes", C.c_int32), ("gene_start", C.POINTER(C.c_int32)),
                ("n_isoforms", C.c_int32), ("n_parts", C.c_int32), ("isoform_start", C.POINTER(C.c_int32)),
                ("part_gene_start", C.POINTER(C.c_int32)), ("n_samples", C.c_int64), ("threshold", C.c_int32),
                ("reserved", C.c_int32), ("device_budget", C.c_uint64)]


class CiStats(C.Structure):
    _fields_ = [("transpose_ms", C.c_double), ("sums_ms", C.c_double), ("sort_ms", C.c_double),
                ("interval_ms", C.c_double), ("blocks", C.c_uint64), ("resident", C.c_int32), ("reserved", C.c_int32)]


class KmerParams(C.Structure):
    _fields_ = [("k", C.c_int32), ("fingerprint_bits", C.c_int32), ("n_transcripts", C.c_uint64),
                ("offsets", C.POINTER(C.c_uint64)), ("bases", C.POINTER(C.c_uint8)), ("max_device_bytes", C.c_uint64)]


class KmerStats(C.Structure):
    _fields_ = [("positions", C.c_uint64), ("table_slots", C.c_uint64), ("input_bytes", C.c_uint64),
                ("table_bytes", C.c_uint64), ("passes", C.c_int32), ("reserved", C.c_int32), ("pack_ms", C.c_double),
                ("insert_ms", C.c_double), ("count_ms", C.c_double)]


class WigBatch(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("n_bytes", C.c_uint64), ("data", C.POINTER(C.c_uint8)),
                ("rec_off", C.POINTER(C.c_uint64)), ("rec_run", C.POINTER(C.c_uint32)), ("run_len", C.POINTER(C.c_uint32)),
                ("n_runs", C.c_uint32), ("continues", C.c_int32), ("keep_last", C.c_int32),
                ("no_fractional_weight", C.c_int32)]


class WigStats(C.Structure):
    _fields_ = [("device_ms", C.c_double), ("blocks", C.c_uint64), ("entries", C.c_uint64), ("bad_record", C.c_int64),
                ("bad_code", C.c_int32), ("reserved", C.c_int32)]


def _dp(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))


def _p(a: Optional[np.ndarray], ct):
    return None if a is None else a.ctypes.data_as(C.POINTER(ct))


def _arr(a, dtype) -> Optional[np.ndarray]:
    if a is None:
        return None
    return np.ascontiguousarray(a, dtype=dtype)


# every symbol include/rsem_b200.h declares (tests check that the .so exports all of them)
SYMBOLS = [
    "rsem_b200_version", "rsem_b200_last_error", "rsem_b200_device_count", "rsem_b200_device_free_bytes",
    "rsem_b200_ctx_create",
    "rsem_b200_ctx_destroy", "rsem_b200_ctx_set_stream", "rsem_b200_ctx_sync", "rsem_b200_ctx_device_bytes",
    "rsem_b200_comm_unique_id", "rsem_b200_comm_init", "rsem_b200_upload_hits", "rsem_b200_upload_conprb",
    "rsem_b200_download_conprb", "rsem_b200_adopt_device_matrix", "rsem_b200_upload_reads", "rsem_b200_upload_refs",
    "rsem_b200_set_model", "rsem_b200_calc_conprb", "rsem_b200_set_theta", "rsem_b200_get_theta",
    "rsem_b200_em_rounds", "rsem_b200_em_model_round", "rsem_b200_expected_weights", "rsem_b200_gibbs_upload",
    "rsem_b200_gibbs_run", "rsem_b200_launch_count", "rsem_b200_estep_timing", "rsem_b200_set_profiling",
    "rsem_b200_set_estep_variant", "rsem_b200_class_layout_info", "rsem_b200_csr_layout_info", "rsem_b200_shard_reads",
    "rsem_b200_estep_cta_times", "rsem_b200_estep_wait_times", "rsem_b200_sim_begin", "rsem_b200_sim_next",
    "rsem_b200_sim_end", "rsem_b200_ci_begin", "rsem_b200_ci_push", "rsem_b200_ci_end", "rsem_b200_kmer_shared",
    "rsem_b200_gbam_convert", "rsem_b200_wig_depth", "rsem_b200_gibbs_run_chains", "rsem_b200_gibbs_sum_chains",
    "rsem_b200_gibbs_split_chains", "rsem_b200_gibbs_upload_from", "rsem_b200_batch_create", "rsem_b200_batch_destroy",
    "rsem_b200_batch_sample_bytes", "rsem_b200_batch_add", "rsem_b200_batch_run", "rsem_b200_batch_slots",
    "rsem_b200_batch_final", "rsem_b200_batch_remove", "rsem_b200_batch_timing", "rsem_b200_gibbs_batch_create",
    "rsem_b200_gibbs_batch_destroy", "rsem_b200_gibbs_batch_sample_bytes", "rsem_b200_gibbs_batch_add",
    "rsem_b200_gibbs_batch_run", "rsem_b200_gibbs_batch_result", "rsem_b200_gibbs_batch_clear",
    "rsem_b200_sim_begin_devices", "rsem_b200_sim_next_devices", "rsem_b200_sim_end_devices", "rsem_b200_mt19937_jump",
    "rsem_b200_sim_upload_refs",
]

RSEM_B200_ERR_ARG = 2
RSEM_B200_ERR_UNSUPPORTED = 4
RSEM_B200_ERR_FULL = 5
GIBBS_BATCH_MIN_READS = 1248
GIBBS_BATCH_MAX_READS = 524288


class Lib:
    def __init__(self, path: str = LIB_PATH):
        if not os.path.exists(path):
            raise RsemB200Error(f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                                "(there is no CPU fallback)")
        self.path = path
        self.dll = C.CDLL(path)
        self.dll.rsem_b200_last_error.restype = C.c_char_p
        for s in SYMBOLS:
            getattr(self.dll, s)  # AttributeError if the library lacks a declared symbol

    def check(self, rc: int):
        if rc != 0:
            raise RsemB200Error(f"librsem_b200 error {rc}: {self.dll.rsem_b200_last_error().decode()}")

    def version(self) -> int:
        return self.dll.rsem_b200_version()

    def device_count(self) -> int:
        n = C.c_int(0)
        self.check(self.dll.rsem_b200_device_count(C.byref(n)))
        return n.value

    def shard_reads(self, row_ptr, n_shards: int):
        """-> [(first_read, last_read_exclusive)] per shard, the reference's thread-sharding rule (EM.cpp:135-157)"""
        row_ptr = _arr(row_ptr, np.uint64)
        bounds = np.zeros(n_shards + 1, np.uint64)
        self.check(self.dll.rsem_b200_shard_reads(C.c_uint64(len(row_ptr) - 1), _p(row_ptr, C.c_uint64), C.c_int32(n_shards),
                                                  _p(bounds, C.c_uint64)))
        return [(int(bounds[i]), int(bounds[i + 1])) for i in range(n_shards)]

    def gibbs_split_chains(self, chain_samples, burnin: int, gap: int, n_parts: int):
        """-> [(first_chain, last_chain_exclusive)] per part: contiguous chain ranges balanced by sweeps"""
        chain_samples = _arr(chain_samples, np.int32)
        bounds = np.zeros(n_parts + 1, np.int32)
        self.check(self.dll.rsem_b200_gibbs_split_chains(C.c_int32(len(chain_samples)), _p(chain_samples, C.c_int32),
                                                         C.c_int32(burnin), C.c_int32(gap), C.c_int32(n_parts),
                                                         _p(bounds, C.c_int32)))
        return [(int(bounds[i]), int(bounds[i + 1])) for i in range(n_parts)]

    def gibbs_sum_chains(self, params: GibbsParams, chain_acc, out: GibbsOut):
        """out's sums = the params.n_chains per-chain blocks of chain_acc added up in chain order"""
        chain_acc = _arr(chain_acc, np.float64)
        self.check(self.dll.rsem_b200_gibbs_sum_chains(C.byref(params), _dp(chain_acc), C.byref(out)))

    def mt19937_jump(self, state, J: int) -> np.ndarray:
        """the boost::mt19937 state (625 uint32: the words, then the index) after J draws from state; host only"""
        state = _arr(state, np.uint32)
        assert state.shape == (625,)
        out = np.zeros(625, np.uint32)
        self.check(self.dll.rsem_b200_mt19937_jump(_p(state, C.c_uint32), C.c_uint64(J), _p(out, C.c_uint32)))
        return out

    def comm_unique_id(self) -> bytes:
        buf = C.create_string_buffer(128)
        self.check(self.dll.rsem_b200_comm_unique_id(buf))
        return buf.raw


_lib: Optional[Lib] = None


def load_library() -> Lib:
    global _lib
    if _lib is None:
        _lib = Lib()
    return _lib


class Context:
    """One GPU context (rsem_b200_ctx).  Methods are 1:1 with the C ABI."""

    def __init__(self, device: int = 0, lib: Optional[Lib] = None):
        self.lib = lib or load_library()
        self._h = C.c_void_p()
        self.lib.check(self.lib.dll.rsem_b200_ctx_create(C.c_int(device), C.byref(self._h)))
        self.N = self.H = self.M = 0
        self._keep = []

    def close(self):
        if self._h:
            self.lib.dll.rsem_b200_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- plumbing
    def set_stream(self, cuda_stream_ptr: int):
        self.lib.check(self.lib.dll.rsem_b200_ctx_set_stream(self._h, C.c_void_p(cuda_stream_ptr)))

    def sync(self):
        self.lib.check(self.lib.dll.rsem_b200_ctx_sync(self._h))

    def device_bytes(self) -> int:
        b = C.c_uint64(0)
        self.lib.check(self.lib.dll.rsem_b200_ctx_device_bytes(self._h, C.byref(b)))
        return b.value

    def comm_init(self, unique_id: bytes, n_ranks: int, rank: int):
        self.lib.check(self.lib.dll.rsem_b200_comm_init(self._h, C.c_char_p(unique_id), n_ranks, rank))

    # ---- data
    def upload_hits(self, row_ptr, sid, M: int, pos=None, insertL=None):
        row_ptr = _arr(row_ptr, np.uint64)
        sid = _arr(sid, np.int32)
        pos = _arr(pos, np.int32)
        insertL = _arr(insertL, np.int32)
        N, H = len(row_ptr) - 1, len(sid)
        self.lib.check(self.lib.dll.rsem_b200_upload_hits(
            self._h, C.c_uint64(N), C.c_uint64(H), C.c_int32(M), _p(row_ptr, C.c_uint64), _p(sid, C.c_int32),
            _p(pos, C.c_int32), _p(insertL, C.c_int32)))
        self.N, self.H, self.M = N, H, M

    def upload_conprb(self, conprb, ncpv):
        conprb, ncpv = _arr(conprb, np.float64), _arr(ncpv, np.float64)
        assert len(conprb) == self.H and len(ncpv) == self.N
        self.lib.check(self.lib.dll.rsem_b200_upload_conprb(self._h, _dp(conprb), _dp(ncpv)))

    def upload_conprb_ptr(self, conprb_ptr: int, ncpv_ptr: int):
        """host pointers (e.g. pinned torch tensors' data_ptr())"""
        self.lib.check(self.lib.dll.rsem_b200_upload_conprb(self._h, C.c_void_p(conprb_ptr), C.c_void_p(ncpv_ptr)))

    def upload_hits_ptr(self, N: int, H: int, M: int, row_ptr_ptr: int, sid_ptr: int):
        self.lib.check(self.lib.dll.rsem_b200_upload_hits(
            self._h, C.c_uint64(N), C.c_uint64(H), C.c_int32(M), C.c_void_p(row_ptr_ptr), C.c_void_p(sid_ptr), None, None))
        self.N, self.H, self.M = N, H, M

    def download_conprb(self):
        conprb, ncpv = np.empty(self.H, np.float64), np.empty(self.N, np.float64)
        self.lib.check(self.lib.dll.rsem_b200_download_conprb(self._h, _dp(conprb), _dp(ncpv)))
        return conprb, ncpv

    def adopt_device_matrix(self, N: int, H: int, M: int, d_row_ptr: int, d_sid: int, d_conprb: int, d_ncpv: int):
        self.lib.check(self.lib.dll.rsem_b200_adopt_device_matrix(
            self._h, C.c_uint64(N), C.c_uint64(H), C.c_int32(M), C.c_void_p(d_row_ptr), C.c_void_p(d_sid),
            C.c_void_p(d_conprb), C.c_void_p(d_ncpv)))
        self.N, self.H, self.M = N, H, M

    def upload_reads(self, off1, base1, qual1, lowq, off2=None, base2=None, qual2=None):
        a = [_arr(off1, np.uint64), _arr(base1, np.uint8), _arr(qual1, np.uint8), _arr(off2, np.uint64),
             _arr(base2, np.uint8), _arr(qual2, np.uint8), _arr(lowq, np.uint8)]
        n_mates = 2 if off2 is not None else 1
        self.lib.check(self.lib.dll.rsem_b200_upload_reads(
            self._h, C.c_int32(n_mates), _p(a[0], C.c_uint64), _p(a[1], C.c_uint8), _p(a[2], C.c_uint8),
            _p(a[3], C.c_uint64), _p(a[4], C.c_uint8), _p(a[5], C.c_uint8), _p(a[6], C.c_uint8)))

    def upload_refs(self, seq_off, seq, full_len, tot_len, mask_off, mask_words):
        a = [_arr(seq_off, np.uint64), _arr(seq, np.uint8), _arr(full_len, np.int32), _arr(tot_len, np.int32),
             _arr(mask_off, np.uint64), _arr(mask_words, np.uint32)]
        M = len(a[2]) - 1
        self.lib.check(self.lib.dll.rsem_b200_upload_refs(
            self._h, C.c_int32(M), _p(a[0], C.c_uint64), _p(a[1], C.c_uint8), _p(a[2], C.c_int32), _p(a[3], C.c_int32),
            _p(a[4], C.c_uint64), _p(a[5], C.c_uint32)))

    def set_model(self, model: Model):
        self.lib.check(self.lib.dll.rsem_b200_set_model(self._h, C.byref(model)))

    # ---- compute
    def calc_conprb(self):
        self.lib.check(self.lib.dll.rsem_b200_calc_conprb(self._h))

    def set_theta(self, theta):
        theta = _arr(theta, np.float64)
        assert len(theta) == self.M + 1
        self.lib.check(self.lib.dll.rsem_b200_set_theta(self._h, _dp(theta)))

    def get_theta(self) -> np.ndarray:
        theta = np.empty(self.M + 1, np.float64)
        self.lib.check(self.lib.dll.rsem_b200_get_theta(self._h, _dp(theta)))
        return theta

    def em_rounds(self, first_round: int, max_rounds: int, min_round: int, max_round: int, n0: float):
        """returns (list of (sum, bchange, totnum), stopped)"""
        stats = (RoundStats * max(max_rounds, 1))()
        ran, stopped = C.c_int32(0), C.c_int32(0)
        self.lib.check(self.lib.dll.rsem_b200_em_rounds(
            self._h, C.c_int32(first_round), C.c_int32(max_rounds), C.c_int32(min_round), C.c_int32(max_round),
            C.c_double(n0), stats, C.byref(ran), C.byref(stopped)))
        return [(stats[i].sum, stats[i].bchange, stats[i].totnum) for i in range(ran.value)], bool(stopped.value)

    def em_model_round(self, n0: float, stats: ModelStats):
        rs = RoundStats()
        self.lib.check(self.lib.dll.rsem_b200_em_model_round(self._h, C.c_double(n0), C.byref(stats), C.byref(rs)))
        return rs.sum, rs.bchange, rs.totnum

    def expected_weights(self) -> np.ndarray:
        counts = np.empty(self.M + 1, np.float64)
        self.lib.check(self.lib.dll.rsem_b200_expected_weights(self._h, _dp(counts)))
        return counts

    def gibbs_upload(self, row_ptr, sid, conprb, M: int):
        row_ptr, sid, conprb = _arr(row_ptr, np.uint64), _arr(sid, np.int32), _arr(conprb, np.float64)
        self.lib.check(self.lib.dll.rsem_b200_gibbs_upload(
            self._h, C.c_uint64(len(row_ptr) - 1), C.c_uint64(len(sid)), C.c_int32(M), _p(row_ptr, C.c_uint64),
            _p(sid, C.c_int32), _dp(conprb)))

    def gibbs_run(self, params: GibbsParams, out: GibbsOut):
        self.lib.check(self.lib.dll.rsem_b200_gibbs_run(self._h, C.byref(params), C.byref(out)))

    def gibbs_run_chains(self, params: GibbsParams, count_vectors: np.ndarray, chain_acc: np.ndarray) -> GibbsStats:
        """count_vectors: int32 (sum of params.chain_samples) x (M + 1); chain_acc: float64, params.n_chains blocks of
        4 (M + 1) + n_genes (both C-contiguous, filled in place)"""
        assert count_vectors.dtype == np.int32 and chain_acc.dtype == np.float64
        assert count_vectors.flags.c_contiguous and chain_acc.flags.c_contiguous
        stats = GibbsStats()
        self.lib.check(self.lib.dll.rsem_b200_gibbs_run_chains(self._h, C.byref(params), _p(count_vectors, C.c_int32),
                                                               _dp(chain_acc), C.byref(stats)))
        return stats

    def gibbs_upload_from(self, src: "Context"):
        """this context gets the matrix uploaded to src (device-to-device copies)"""
        self.lib.check(self.lib.dll.rsem_b200_gibbs_upload_from(self._h, src._h if src is not None else None))

    def sim_upload_refs(self, seq_off: np.ndarray, seq: np.ndarray, tot_len: np.ndarray, full_len: np.ndarray):
        """keeps the reference on the context (M = len(tot_len) - 1): a following sim_begin whose params.seq is NULL
        uses it"""
        seq_off, seq = _arr(seq_off, np.uint64), _arr(seq, np.uint8)
        tot_len, full_len = _arr(tot_len, np.int32), _arr(full_len, np.int32)
        self.lib.check(self.lib.dll.rsem_b200_sim_upload_refs(self._h, C.c_int32(len(tot_len) - 1), _p(seq_off, C.c_uint64),
                                                              _p(seq, C.c_uint8), _p(tot_len, C.c_int32),
                                                              _p(full_len, C.c_int32)))

    def sim_begin(self, params: SimParams):
        """params' arrays must stay alive until sim_begin returns (they are copied to the device)"""
        self.lib.check(self.lib.dll.rsem_b200_sim_begin(self._h, C.byref(params)))

    def sim_next(self):
        """-> (n_reads, [mate 1 text, mate 2 text]) of the next chunk; n_reads == 0 after the last one"""
        text = (C.c_void_p * 2)()
        nbytes = (C.c_uint64 * 2)()
        n = C.c_uint64(0)
        self.lib.check(self.lib.dll.rsem_b200_sim_next(self._h, text, nbytes, C.byref(n)))
        return n.value, [C.string_at(text[i], nbytes[i]) if text[i] else b"" for i in range(2)]

    def sim_end(self, M: int):
        """-> (counts per sid, M + 1 doubles; number of failed attempts; SimStats phase times)"""
        counts = np.zeros(M + 1, np.float64)
        resim = C.c_uint64(0)
        stats = SimStats()
        self.lib.check(self.lib.dll.rsem_b200_sim_end(self._h, _dp(counts), C.byref(resim), C.byref(stats)))
        return counts, resim.value, stats

    def ci_begin(self, params: CiParams):
        """params' arrays must stay alive until ci_begin returns (they are copied)"""
        self.lib.check(self.lib.dll.rsem_b200_ci_begin(self._h, C.byref(params)))

    def ci_push(self, rows, l_bars, first: int):
        """rows: count x M float32 TPMs of samples first .. first + count - 1, l_bars: their count mean lengths"""
        rows, l_bars = _arr(rows, np.float32), _arr(l_bars, np.float32)
        self.lib.check(self.lib.dll.rsem_b200_ci_push(self._h, _p(rows, C.c_float), _p(l_bars, C.c_float),
                                                      C.c_int64(first), C.c_int64(len(l_bars))))

    def ci_end(self, M: int, n_genes: int, n_isoforms: int = 0):
        """-> (transcripts M x 6, genes n_genes x 6, isoforms n_isoforms x 6, CiStats); columns are the TPM lb, ub, cqv
        and the FPKM lb, ub, cqv"""
        tr = np.zeros((M, 6), np.float32)
        ge = np.zeros((n_genes, 6), np.float32)
        iso = np.zeros((n_isoforms, 6), np.float32)
        stats = CiStats()
        self.lib.check(self.lib.dll.rsem_b200_ci_end(self._h, _p(tr, C.c_float), _p(ge, C.c_float),
                                                     _p(iso, C.c_float) if n_isoforms else None, C.byref(stats)))
        return tr, ge, iso, stats

    def kmer_shared(self, k: int, offsets, bases, max_device_bytes: int = 0, fingerprint_bits: int = 0):
        """-> (per transcript, the start positions whose k-mer also starts in another transcript, uint64; KmerStats).
        offsets: n + 1 transcript offsets into bases, codes 0..4 (A C G T N)"""
        offsets, bases = _arr(offsets, np.uint64), _arr(bases, np.uint8)
        n = len(offsets) - 1
        counts = np.zeros(max(n, 1), np.uint64)
        params = KmerParams(k=k, fingerprint_bits=fingerprint_bits, n_transcripts=n, offsets=_p(offsets, C.c_uint64),
                            bases=_p(bases, C.c_uint8), max_device_bytes=max_device_bytes)
        stats = KmerStats()
        self.lib.check(self.lib.dll.rsem_b200_kmer_shared(self._h, C.byref(params), _p(counts, C.c_uint64),
                                                          C.byref(stats)))
        return counts[:n], stats

    def wig_depth(self, data, rec_off, rec_run, run_len, continues: bool = False, keep_last: bool = False,
                  no_fractional_weight: bool = False, out_len: Optional[int] = None):
        """one call of K11 -> (the depth arrays of the runs it finished, concatenated; WigStats).  data: mapped records,
        each after its u32 block_size, at rec_off; rec_run: each record's run; run_len: each run's target length.
        out_len: room for the output (default: the batch's positions plus any resident run's, as the caller knows)"""
        data = _arr(np.frombuffer(bytes(data), np.uint8) if isinstance(data, (bytes, bytearray)) else data, np.uint8)
        rec_off, rec_run, run_len = _arr(rec_off, np.uint64), _arr(rec_run, np.uint32), _arr(run_len, np.uint32)
        cap = int(run_len.sum()) if out_len is None else out_len
        out = np.zeros(max(cap, 1), np.float64)
        b = WigBatch(n_records=len(rec_off), n_bytes=len(data), data=_p(data, C.c_uint8), rec_off=_p(rec_off, C.c_uint64),
                     rec_run=_p(rec_run, C.c_uint32), run_len=_p(run_len, C.c_uint32), n_runs=len(run_len),
                     continues=int(continues), keep_last=int(keep_last), no_fractional_weight=int(no_fractional_weight))
        got = C.c_uint64(0)
        stats = WigStats()
        self.lib.check(self.lib.dll.rsem_b200_wig_depth(self._h, C.byref(b), _dp(out), C.c_uint64(cap), C.byref(got),
                                                        C.byref(stats)))
        return out[: got.value], stats

    # ---- instrumentation
    def launch_count(self) -> int:
        n = C.c_uint64(0)
        self.lib.check(self.lib.dll.rsem_b200_launch_count(self._h, C.byref(n)))
        return n.value

    def estep_timing(self, reset: bool = False):
        ms, n = C.c_double(0), C.c_uint64(0)
        self.lib.check(self.lib.dll.rsem_b200_estep_timing(self._h, C.byref(ms), C.byref(n), C.c_int32(int(reset))))
        return ms.value, n.value

    def set_profiling(self, on: bool):
        self.lib.check(self.lib.dll.rsem_b200_set_profiling(self._h, C.c_int32(int(on))))

    def class_layout_info(self) -> dict:
        out = (C.c_uint64 * 10)()
        self.lib.check(self.lib.dll.rsem_b200_class_layout_info(self._h, out))
        keys = ("built", "rows", "long_rows", "segments", "batches", "tiles", "vals", "ids", "tiles_main", "run_hits")
        d = dict(zip(keys, (int(x) for x in out)))
        d["bytes_per_round"] = 8 * d["vals"] + 4 * d["ids"] + 16 * d["batches"]
        return d

    def csr_layout_info(self) -> dict:
        out = (C.c_uint64 * 6)()
        self.lib.check(self.lib.dll.rsem_b200_csr_layout_info(self._h, out))
        keys = ("tiles", "tile_weight", "rows_group", "group", "max_deg", "has_empty")
        return dict(zip(keys, (int(x) for x in out)))

    def estep_cta_times(self) -> np.ndarray:
        out = np.zeros(1024, np.uint64)
        n = C.c_int32(0)
        self.lib.check(self.lib.dll.rsem_b200_estep_cta_times(self._h, _p(out, C.c_uint64), C.c_int32(1024), C.byref(n)))
        return out[: n.value]

    def estep_wait_times(self) -> np.ndarray:
        """per CTA of the latest profiled class-kernel launch: (consumer ns blocked on data summed over its warps,
        copy-issuer ns blocked on a free stage, consumer warps, SM cycles summed over the consumer warps in the phases
        front, rows, flush and hand-over, SM cycles the CTA was busy); empty when that launch ran without profiling"""
        out = np.zeros((1024, 8), np.uint64)
        n = C.c_int32(0)
        self.lib.check(self.lib.dll.rsem_b200_estep_wait_times(self._h, _p(out, C.c_uint64), C.c_int32(1024), C.byref(n)))
        return out[: n.value]

    def set_estep_variant(self, v: int):
        self.lib.check(self.lib.dll.rsem_b200_set_estep_variant(self._h, C.c_int32(v)))


class SimDevices:
    """rsem-simulate-reads over several contexts (rsem_b200_sim_*_devices): the reads of Context.sim_* on one context"""

    def __init__(self, ctxs, params: SimParams):
        """params' arrays must stay alive until the constructor returns (they are copied to the devices)"""
        self.lib = ctxs[0].lib
        self.ctxs = list(ctxs)
        self._h = C.c_void_p()
        arr = (C.c_void_p * len(ctxs))(*[c._h.value for c in ctxs])
        self.lib.check(self.lib.dll.rsem_b200_sim_begin_devices(arr, C.c_int(len(ctxs)), C.byref(params), C.byref(self._h)))

    def next(self):
        """-> (n_reads, [mate 1 text, mate 2 text]) of the next chunk; n_reads == 0 after the last one"""
        text = (C.c_void_p * 2)()
        nbytes = (C.c_uint64 * 2)()
        n = C.c_uint64(0)
        self.lib.check(self.lib.dll.rsem_b200_sim_next_devices(self._h, text, nbytes, C.byref(n)))
        return n.value, [C.string_at(text[i], nbytes[i]) if text[i] else b"" for i in range(2)]

    def end(self, M: int):
        """-> (counts per sid, M + 1 doubles; failed attempts; SimDevicesStats; [SimStats per context])"""
        counts = np.zeros(M + 1, np.float64)
        resim = C.c_uint64(0)
        stats = SimDevicesStats()
        per = (SimStats * len(self.ctxs))()
        h, self._h = self._h, C.c_void_p()
        self.lib.check(self.lib.dll.rsem_b200_sim_end_devices(h, _dp(counts), C.byref(resim), C.byref(stats), per))
        return counts, resim.value, stats, list(per)


class Batch:
    """K12: the frozen-conprb rounds of many samples in one device arena (include/rsem_b200.h, rsem_b200_batch_*)."""

    def __init__(self, ctx: Context, capacity_bytes: int = 0):
        self.lib = ctx.lib
        self.ctx = ctx   # the batch lives on the context's device and stream
        self._h = C.c_void_p()
        self.lib.check(self.lib.dll.rsem_b200_batch_create(ctx._h, C.c_uint64(capacity_bytes), C.byref(self._h)))
        self.shapes = {}

    def close(self):
        if self._h:
            self.lib.dll.rsem_b200_batch_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def sample_bytes(self, row_ptr, m: int) -> int:
        row_ptr = _arr(row_ptr, np.uint64)
        out = C.c_uint64(0)
        self.lib.check(self.lib.dll.rsem_b200_batch_sample_bytes(
            C.c_uint64(len(row_ptr) - 1), C.c_uint64(int(row_ptr[-1])), _p(row_ptr, C.c_uint64), C.c_int32(m),
            C.byref(out)))
        return out.value

    def add(self, row_ptr, sid, conprb, ncpv, theta, n0: float, first_round: int, min_round: int, max_round: int) -> int:
        """returns the slot; raises RsemB200Error (code RSEM_B200_ERR_FULL in .code) when the arena is full"""
        row_ptr, sid = _arr(row_ptr, np.uint64), _arr(sid, np.int32)
        conprb, ncpv, theta = _arr(conprb, np.float64), _arr(ncpv, np.float64), _arr(theta, np.float64)
        N, H, M = len(row_ptr) - 1, len(sid), len(theta) - 1
        slot = C.c_int32(-1)
        rc = self.lib.dll.rsem_b200_batch_add(
            self._h, C.c_uint64(N), C.c_uint64(H), C.c_int32(M), _p(row_ptr, C.c_uint64), _p(sid, C.c_int32),
            _dp(conprb), _dp(ncpv), _dp(theta), C.c_double(n0), C.c_int32(first_round), C.c_int32(min_round),
            C.c_int32(max_round), C.byref(slot))
        if rc != 0:
            err = RsemB200Error(f"librsem_b200 error {rc}: {self.lib.dll.rsem_b200_last_error().decode()}")
            err.code = rc
            raise err
        self.shapes[slot.value] = (N, H, M)
        return slot.value

    def run(self, max_rounds: int):
        """one launch; returns {slot: (list of (sum, bchange, totnum), stopped)}"""
        n = C.c_int32(0)
        self.lib.check(self.lib.dll.rsem_b200_batch_slots(self._h, C.byref(n)))
        k = max(max_rounds, 1)
        stats = (RoundStats * (max(n.value, 1) * k))()
        ran = np.zeros(max(n.value, 1), np.int32)
        stopped = np.zeros(max(n.value, 1), np.int32)
        self.lib.check(self.lib.dll.rsem_b200_batch_run(self._h, C.c_int32(max_rounds), stats, _p(ran, C.c_int32),
                                                        _p(stopped, C.c_int32)))
        return {s: ([(stats[s * k + r].sum, stats[s * k + r].bchange, stats[s * k + r].totnum) for r in range(ran[s])],
                    bool(stopped[s])) for s in self.shapes}

    def final(self, slot: int, posteriors: bool = False):
        """(theta M + 1, counts M + 1 without N0, post H or None, post0 N or None)"""
        N, H, M = self.shapes[slot]
        theta, counts = np.empty(M + 1), np.empty(M + 1)
        post = np.empty(max(H, 1)) if posteriors else None
        post0 = np.empty(N) if posteriors else None
        self.lib.check(self.lib.dll.rsem_b200_batch_final(self._h, C.c_int32(slot), _dp(theta), _dp(counts), _dp(post),
                                                          _dp(post0)))
        return theta, counts, (post[:H] if posteriors else None), post0

    def remove(self, slot: int):
        self.lib.check(self.lib.dll.rsem_b200_batch_remove(self._h, C.c_int32(slot)))
        del self.shapes[slot]

    def timing(self):
        """(K12 device ms summed over launches, sample-rounds run)"""
        ms, n = C.c_double(0), C.c_uint64(0)
        self.lib.check(self.lib.dll.rsem_b200_batch_timing(self._h, C.byref(ms), C.byref(n)))
        return ms.value, n.value


class GibbsBatch:
    """K13: the Gibbs chains of many samples in one cooperative launch (include/rsem_b200.h, rsem_b200_gibbs_batch_*)."""

    def __init__(self, ctx: Context, capacity_bytes: int = 0, worker_ctas: int = 0):
        self.lib = ctx.lib
        self.ctx = ctx   # the batch lives on the context's device and stream
        self._h = C.c_void_p()
        self.lib.check(self.lib.dll.rsem_b200_gibbs_batch_create(ctx._h, C.c_uint64(capacity_bytes), C.c_int32(worker_ctas),
                                                                 C.byref(self._h)))
        self.shapes = {}

    def close(self):
        if self._h:
            self.lib.dll.rsem_b200_gibbs_batch_destroy(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def sample_bytes(self, N1: int, E: int, M: int, n_genes: int, n_samples: int, n_chains: int) -> int:
        out = C.c_uint64(0)
        self.lib.check(self.lib.dll.rsem_b200_gibbs_batch_sample_bytes(
            C.c_uint64(N1), C.c_uint64(E), C.c_int32(M), C.c_int32(n_genes), C.c_int32(n_samples), C.c_int32(n_chains),
            C.byref(out)))
        return out.value

    def add(self, row_ptr, sid, conprb, params: GibbsParams) -> int:
        """returns the slot; raises RsemB200Error with .code (RSEM_B200_ERR_FULL, RSEM_B200_ERR_UNSUPPORTED, ...)"""
        row_ptr, sid, conprb = _arr(row_ptr, np.uint64), _arr(sid, np.int32), _arr(conprb, np.float64)
        slot = C.c_int32(-1)
        rc = self.lib.dll.rsem_b200_gibbs_batch_add(self._h, C.c_uint64(len(row_ptr) - 1), C.c_uint64(len(sid)),
                                                    _p(row_ptr, C.c_uint64), _p(sid, C.c_int32), _dp(conprb),
                                                    C.byref(params), C.byref(slot))
        if rc != 0:
            err = RsemB200Error(f"librsem_b200 error {rc}: {self.lib.dll.rsem_b200_last_error().decode()}")
            err.code = rc
            raise err
        samples = [params.chain_samples[t] for t in range(params.n_chains)]
        self.shapes[slot.value] = (params.M, params.n_genes, samples)
        return slot.value

    def run(self) -> GibbsBatchStats:
        stats = GibbsBatchStats()
        self.lib.check(self.lib.dll.rsem_b200_gibbs_batch_run(self._h, C.byref(stats)))
        return stats

    def result(self, slot: int):
        """(count vectors: int32 sum(chain_samples) x (M + 1), chain_acc: float64 n_chains x (4 (M + 1) + n_genes))"""
        M, n_genes, samples = self.shapes[slot]
        cv = np.zeros((sum(samples), M + 1), np.int32)
        acc = np.zeros((len(samples), 4 * (M + 1) + n_genes))
        self.lib.check(self.lib.dll.rsem_b200_gibbs_batch_result(self._h, C.c_int32(slot), _p(cv, C.c_int32), _dp(acc)))
        return cv, acc

    def clear(self):
        self.lib.check(self.lib.dll.rsem_b200_gibbs_batch_clear(self._h))
        self.shapes = {}
