"""ctypes binding of libmpb200.so (include/mpb200.h).  No CPU fallback: every compute call needs an H100."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libmpb200.so")

MAX_K = 27
KEY_EMPTY = 0xFFFFFFFFFFFFFFFF
KEY_IUPAC = 0xFFFFFFFFFFFFFFFE
KEY_BASE5 = 1 << 54

_lib = None

# name -> (restype, argtypes); mirrors include/mpb200.h one to one
_P = C.c_void_p
SIGNATURES = {
    "mpb_abi_version": (C.c_int, []),
    "mpb_last_error": (C.c_char_p, []),
    "mpb_device_count": (C.c_int, []),
    "mpb_ctx_create": (C.c_int, [C.c_int, C.POINTER(_P)]),
    "mpb_ctx_destroy": (None, [_P]),
    "mpb_ctx_set_stream": (C.c_int, [_P, _P]),
    "mpb_ctx_sync": (C.c_int, [_P]),
    "mpb_ctx_launches": (C.c_int64, [_P]),
    "mpb_ctx_memcpy": (C.c_int, [_P, _P, _P, C.c_int64]),
    "mpb_ctx_memset": (C.c_int, [_P, _P, C.c_int, C.c_int64]),
    "mpb_dev_alloc": (C.c_int, [_P, C.c_int64, C.POINTER(_P)]),
    "mpb_dev_free": (None, [_P, _P]),
    "mpb_ctx_profile": (C.c_int, [_P, C.c_int]),
    "mpb_ctx_profile_read": (C.c_int, [_P, C.c_char_p, C.POINTER(C.c_double), C.POINTER(C.c_int64),
                                        C.POINTER(C.c_double)]),
    "mpb_msa_upload": (C.c_int, [_P, _P, C.c_int64, C.c_int64, C.c_int64, _P, C.POINTER(_P)]),
    "mpb_msa_free": (None, [_P]),
    "mpb_msa_nseq": (C.c_int64, [_P]),
    "mpb_msa_set_row0": (C.c_int, [_P, C.c_int64]),
    "mpb_hist_counts": (C.c_int, [_P, _P, _P, _P]),
    "mpb_hist_export": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "mpb_seq_attr": (C.c_int, [_P, _P, _P]),
    "mpb_seq_attr_hist": (C.c_int, [_P, _P, _P]),
    "mpb_window_prefilter": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int32, _P, _P]),
    "mpb_hist_build": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int32, C.c_int, C.POINTER(_P)]),
    "mpb_hist_free": (None, [_P]),
    "mpb_hist_merge": (C.c_int, [_P, _P, _P, _P, _P]),
    "mpb_hist_stats": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P]),
    "mpb_hist_tensors": (C.c_int, [_P, _P, _P, _P]),
    "mpb_hist_dump": (C.c_int, [_P, C.c_int32, C.c_int64, _P, _P, _P, C.POINTER(C.c_int64)]),
    "mpb_hist_match": (C.c_int, [_P, _P, _P, C.c_int32, _P]),
    "mpb_hist_exceptions": (C.c_int, [_P, C.c_int64, _P, _P, C.POINTER(C.c_int64)]),
    "mpb_scan": (C.c_int, [_P, C.c_int, C.c_int, C.c_uint32, C.c_uint32, _P, _P, C.c_int64, _P, _P, _P]),
    "mpb_pattern_hits": (C.c_int, [_P, C.c_int32, _P, _P, C.c_int64, _P, _P, _P, C.POINTER(C.c_int64)]),
    "mpb_pattern_sites": (C.c_int, [_P, C.c_int32, _P, _P, _P, C.c_int32, C.c_int64, _P, _P, _P, _P,
                                    C.POINTER(C.c_int64)]),
    "mpb_pattern_products": (C.c_int, [_P, C.c_int32, _P, _P, _P, C.c_int32, _P, _P, C.c_int32, C.c_int64, C.c_int32,
                                       _P, _P, C.c_int32, C.c_int32, _P, C.c_int64, C.c_int64, _P, _P, _P,
                                       C.POINTER(C.c_int64), _P]),
    "mpb_seqkeys": (C.c_int, [_P, C.c_int, _P, C.c_int32, _P]),
    "mpb_tm": (C.c_int, [_P, _P, C.c_int, C.c_int64, _P, _P, _P, _P]),
    "mpb_tm_sets": (C.c_int, [_P, _P, C.c_int, C.c_int32, _P, _P, _P]),
    "mpb_walk": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int32, _P, _P, _P, _P, _P, _P,
                           _P, _P, _P, _P, _P, C.c_int64, _P, _P, _P]),
    "mpb_hist_export_at": (C.c_int, [_P, C.c_int32, _P, _P, _P, C.c_int64, _P, _P, _P]),
    "mpb_hist_merge_segments": (C.c_int, [_P, C.c_int32, _P, _P, _P, _P]),
    "mpb_hist_create_empty": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int32, C.c_int, C.POINTER(_P)]),
    "mpb_hist_add_counts": (C.c_int, [_P, _P, _P]),
    "mpb_hist_summary": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "mpb_cscan": (C.c_int, [_P, C.c_uint32, C.c_uint32, _P, C.c_int64, _P, _P, _P]),
    "mpb_walk_dev_begin": (C.c_int, [_P, C.c_int, C.c_int, C.c_uint32, C.c_uint32, C.c_int32, _P, _P, _P, _P, _P,
                                      C.POINTER(_P)]),
    "mpb_walk_dev_advance": (C.c_int, [_P]),
    "mpb_walk_dev_scan": (C.c_int, [_P]),
    "mpb_walk_dev_round": (C.c_int, [_P]),
    "mpb_walk_dev_counts": (C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_int64)]),
    "mpb_walk_dev_live": (C.c_int64, [_P]),
    "mpb_walk_dev_max_rounds": (C.c_int, [_P]),
    "mpb_walk_dev_wait": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int64)]),
    "mpb_walk_dev_run": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int64)]),
    "mpb_walk_dev_finish": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int64, _P, _P, _P]),
    "mpb_walk_dev_free": (None, [_P]),
    "mpb_walk_dev_set_peer": (C.c_int, [_P, _P]),
    "mpb_peer_create": (C.c_int, [_P, C.c_int, C.c_int, C.c_int64, C.POINTER(_P)]),
    "mpb_peer_handle": (C.c_int, [_P, _P]),
    "mpb_peer_connect": (C.c_int, [_P, _P]),
    "mpb_peer_cap": (C.c_int64, [_P]),
    "mpb_peer_allreduce": (C.c_int, [_P, _P, C.c_int64]),
    "mpb_peer_allreduce_phases": (C.c_int, [_P, _P, C.c_int64, C.c_int]),
    "mpb_peer_free": (None, [_P]),
    "mpb_primer_props": (C.c_int, [_P, _P, C.c_int, C.c_int32, C.c_double, C.c_double, C.c_int, _P, _P, _P, _P, _P,
                                   _P]),
    "mpb_window_cells": (C.c_int, [_P, C.c_int64, _P, C.c_int32, C.c_int, C.c_int64, _P, _P, _P, _P]),
    "mpb_pair_cover": (C.c_int, [_P, _P, _P, C.c_int32, C.c_int32, _P, _P, C.c_int64, _P]),
    "mpb_pair_cover3": (C.c_int, [_P, _P, C.c_int32, C.c_int64, _P, _P, C.c_int64, _P]),
    "mpb_dimer_prepare": (C.c_int, [_P, _P, _P, C.c_int32, C.c_int, C.c_int, C.c_int, _P, _P, C.POINTER(_P)]),
    "mpb_dimer_free": (None, [_P]),
    "mpb_dimer_counts": (C.c_int, [_P, _P, _P]),
    "mpb_dimer_pairs": (C.c_int, [_P, _P, _P, C.c_int64, _P, _P]),
    "mpb_dimer_grid": (C.c_int, [_P, C.c_int32, C.c_int32, C.c_int64, _P, _P, _P, _P, C.POINTER(C.c_int64),
                                  C.POINTER(C.c_int64)]),
    "mpb_pool_search": (C.c_int, [_P, C.c_int32, C.c_int32, _P, C.c_uint64, C.c_int64, C.c_int64, C.c_int32, _P, _P,
                                  _P]),
    "mpb_pattern_cover": (C.c_int, [_P, C.c_int32, _P, _P, _P, C.c_int32, C.c_int64, C.c_int32, _P, _P, C.c_int32,
                                    C.c_int32, C.c_int64, _P, _P, C.c_int64, _P]),
    "mpb_cover_gains": (C.c_int, [_P, _P, _P, C.c_int64, C.c_int64, _P, _P, _P, C.c_int64, _P]),
    "mpb_cover_take": (C.c_int, [_P, _P, _P, C.c_int64, C.c_int64, C.c_int64, _P, _P]),
    "mpb_site_list_create": (C.c_int, [_P, C.c_int32, _P, C.c_int64, C.c_int32, _P, _P, C.POINTER(_P)]),
    "mpb_site_list_destroy": (None, [_P]),
    "mpb_pattern_cover_keep": (C.c_int, [_P, C.c_int32, _P, _P, _P, C.c_int32, C.c_int64, C.c_int32, _P, _P, C.c_int32,
                                         C.c_int32, C.c_int64, _P, _P, C.c_int64, _P, _P, C.c_int32]),
    "mpb_site_list_seal": (C.c_int, [_P, C.POINTER(C.c_int64)]),
    "mpb_site_list_keys": (C.c_int, [_P, C.c_int64, _P, C.POINTER(C.c_int64)]),
    "mpb_sites_cross": (C.c_int, [_P, C.c_int32, C.c_int32, C.c_int32, _P, _P]),
    "mpb_sites_own": (C.c_int, [_P, C.c_int32, C.c_int32, _P]),
}


SCAN_CB = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64))
CAND_DTYPE = np.dtype([("win", np.int32), ("trial", np.int32), ("allow", np.uint32, (4,))])     # struct mpb_cand


class MpbError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__("libmpb200 error %d: %s" % (code, msg))
        self.code = code


def load():
    """dlopen libmpb200.so (building it is build.py's job; a missing library is an error, not a fallback)"""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError("libmpb200.so is missing: run `python -m multiprime_b200.build` (needs nvcc)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    if lib.mpb_abi_version() != 3:
        raise ImportError("libmpb200.so ABI version mismatch")
    _lib = lib
    return lib


def check(rc: int):
    if rc != 0:
        raise MpbError(rc, load().mpb_last_error().decode())


def ptr(x):
    """numpy array / torch tensor / int / None -> void*"""
    if x is None:
        return None
    if isinstance(x, np.ndarray):
        assert x.flags["C_CONTIGUOUS"]
        return x.ctypes.data_as(C.c_void_p)
    if hasattr(x, "data_ptr"):
        return C.c_void_p(x.data_ptr())
    return C.c_void_p(int(x))


def window_cells(packed4: np.ndarray, lens, n_col: int, k: int, seq, pos):
    """mpb_window_cells: raw k-mers (core:666-687) of (sequence, window) pairs from the host copy of the alignment
    -> (cells uint8[n, 32], length int32[n]).  Pure host code."""
    assert packed4.dtype == np.uint8 and packed4.flags.c_contiguous and packed4.ndim == 2
    seq = np.ascontiguousarray(seq, dtype=np.int64)
    pos = np.ascontiguousarray(pos, dtype=np.int32)
    lens = None if lens is None else np.ascontiguousarray(lens, dtype=np.int32)
    n = len(seq)
    cells = np.zeros((n, 32), np.uint8)
    out_len = np.zeros(n, np.int32)
    if n:
        if seq.min() < 0 or seq.max() >= packed4.shape[0]:
            raise IndexError("sequence index outside the alignment")
        check(load().mpb_window_cells(ptr(packed4), packed4.shape[1], ptr(lens), n_col, k, n, ptr(seq), ptr(pos),
                                      ptr(cells), ptr(out_len)))
    return cells, out_len


def make_cands(win, allow, trial=None) -> np.ndarray:
    """struct mpb_cand array from window indices, allowed-base masks [n, 4] and optional trial codes"""
    win = np.asarray(win, dtype=np.int32)
    c = np.zeros(len(win), CAND_DTYPE)
    c["win"] = win
    c["allow"] = np.asarray(allow, dtype=np.uint32).reshape(-1, 4)
    c["trial"] = -1 if trial is None else np.asarray(trial, dtype=np.int32)
    return c


def _walk_outputs(n):
    return dict(sets=np.zeros((n, 32), np.uint8), counts=np.zeros((n, 5), np.int64), seeds=np.zeros((n, 2, 32), np.uint8),
                seed_cover=np.zeros((n, 2), np.int64), ntracks=np.zeros(n, np.int32), stats=np.zeros(3, np.int64))


def walk(k, v, dnum, degeneracy, cover_number, freq, nn, mm_key, scan_fn, want_trace=True):
    """mpb_walk: refinement walk of a window batch on the HOST; scan_fn(cands: CAND_DTYPE[nc]) -> int64[nc,4]
    (perfect, F_mis, R_mis, trial perfect); candidates name windows 0..n-1.  No CUDA calls: the CPU tests drive it
    with a stand-in scan; the GPU path is WalkDev."""
    n = len(cover_number)
    cover_number = np.ascontiguousarray(cover_number, dtype=np.int64)
    freq = np.ascontiguousarray(freq, dtype=np.int64)
    nn = np.ascontiguousarray(nn, dtype=np.int64)
    mm_key = np.ascontiguousarray(mm_key, dtype=np.uint64)
    err = []

    def cb(_user, p_cands, nc, p_counts):
        try:
            cands = np.ctypeslib.as_array(C.cast(p_cands, C.POINTER(C.c_uint8)), shape=(nc * CAND_DTYPE.itemsize,))
            out = np.ctypeslib.as_array(p_counts, shape=(nc, 4))
            out[:] = scan_fn(cands.view(CAND_DTYPE))
            return 0
        except Exception as exc:           # surfaced after mpb_walk returns
            err.append(exc)
            return -2

    res = _walk_outputs(n)
    cap = max(64, n * 48)
    cfn = SCAN_CB(cb)
    while True:
        trace = np.zeros((cap, 32), np.uint8)
        off = np.zeros(n + 1, np.int64)
        rc = load().mpb_walk(k, v, dnum, degeneracy, n, ptr(cover_number), ptr(freq), ptr(nn), ptr(mm_key),
                             C.cast(cfn, C.c_void_p), None, ptr(res["sets"]), ptr(res["counts"]), ptr(res["seeds"]),
                             ptr(res["seed_cover"]), ptr(res["ntracks"]), cap, ptr(trace), ptr(off), ptr(res["stats"]))
        if err:
            raise err[0]
        if rc == -4 and res["stats"][2] > cap:      # trace buffer too small: the walk is deterministic, run it again
            cap = int(res["stats"][2]) + 16
            continue
        check(rc)
        break
    res.update(trace=trace, trace_off=off)
    return res


class DevBuf:
    """caller-owned device memory (mpb_dev_alloc): results that stay in HBM between calls"""

    def __init__(self, ctx: "Context", shape, dtype):
        self.ctx, self.shape, self.dtype = ctx, tuple(int(x) for x in shape), np.dtype(dtype)
        self.nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        p = C.c_void_p()
        check(load().mpb_dev_alloc(ctx.h, self.nbytes, C.byref(p)))
        self.p = p.value

    def data_ptr(self) -> int:          # ptr() takes anything with data_ptr()
        return self.p

    def at(self, index: int) -> int:
        """device address of element [index] along the first axis"""
        return self.p + index * (self.nbytes // max(1, self.shape[0]))

    def to_host(self) -> np.ndarray:
        out = np.empty(self.shape, self.dtype)
        check(load().mpb_ctx_memcpy(self.ctx.h, ptr(out), C.c_void_p(self.p), self.nbytes))
        return out

    def zero(self):
        check(load().mpb_ctx_memset(self.ctx.h, C.c_void_p(self.p), 0, self.nbytes))

    def close(self):
        if self.p and self.ctx.h:
            load().mpb_dev_free(self.ctx.h, C.c_void_p(self.p))
        self.p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CoverMatrix:
    """mpb_pattern_cover's bits in HBM: amp / perf [n_rows, words] (bit r of row c set when pair c amplifies record r /
    has a perfect amplicon there) and the covered / covered_perfect vectors of a greedy over them, all zeroed at the
    start.  words = ceil(n_rec / 128) * 4 (at least 4): rows are whole 128-bit loads."""

    def __init__(self, ctx: "Context", n_rows: int, n_rec: int):
        self.ctx, self.n_rows, self.n_rec = ctx, int(n_rows), int(n_rec)
        self.words = words_of(n_rec)
        self.buf = DevBuf(ctx, (2 * self.n_rows + 2, self.words), np.uint32)     # amp rows, perf rows, the two vectors
        try:
            self.buf.zero()
        except MpbError:
            self.buf.close()
            raise
        self.amp, self.perf = self.buf.at(0), self.buf.at(self.n_rows)
        self.covered, self.covered_perfect = self.buf.at(2 * self.n_rows), self.buf.at(2 * self.n_rows + 1)

    def to_host(self):
        """(amp, perf, covered, covered_perfect) as uint32 arrays"""
        a = self.buf.to_host()
        n = self.n_rows
        return a[:n], a[n:2 * n], a[2 * n], a[2 * n + 1]

    def close(self):
        self.buf.close()


class SiteList:
    """mpb_site_list: the filtered sites of a panel's n_pat patterns (lens[n_pat]) over the records rec_off / rec_len of
    a stream of n_pos columns, kept in HBM by Msa.pattern_cover_keep, sealed once, then joined (cross / own)"""

    def __init__(self, ctx: "Context", lens, n_pos: int, rec_off, rec_len):
        self.ctx = ctx
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        rec_off = np.ascontiguousarray(rec_off, dtype=np.int64)
        rec_len = np.ascontiguousarray(rec_len, dtype=np.int64)
        self.n_pairs = len(lens) // 4
        h = C.c_void_p()
        check(load().mpb_site_list_create(ctx.h, len(lens), ptr(lens), int(n_pos), len(rec_off), ptr(rec_off),
                                          ptr(rec_len), C.byref(h)))
        self.h = h

    def seal(self) -> int:
        """sort the kept sites into stream order -> their number"""
        n = C.c_int64()
        check(load().mpb_site_list_seal(self.h, C.byref(n)))
        return n.value

    def keys(self) -> np.ndarray:
        """the list's keys (position << (bits(n_pat) + 4) | pattern << 4 | mismatches) in list order"""
        n = C.c_int64()
        check(load().mpb_site_list_keys(self.h, 0, None, C.byref(n)))
        out = np.zeros(n.value, np.uint64)
        check(load().mpb_site_list_keys(self.h, len(out), ptr(out), C.byref(n)))
        return out

    def cross(self, lo: int, hi: int, pair: int, eligible) -> np.ndarray:
        """mpb_sites_cross -> uint8[pairs]: the products between pair `pair` and the pairs flagged in eligible
        (bool[pairs]), bit side << 2 | primer of the pair << 1 | primer of `pair`"""
        el = np.packbits(np.asarray(eligible, bool), bitorder="little")
        el = np.ascontiguousarray(np.pad(el, (0, -len(el) % 4)).view(np.uint32))
        out = np.zeros(self.n_pairs, np.uint8)
        check(load().mpb_sites_cross(self.h, lo, hi, int(pair), ptr(el), ptr(out)))
        return out

    def own(self, lo: int, hi: int) -> np.ndarray:
        """mpb_sites_own -> uint8[pairs]: bit left primer << 1 | right primer when the pair's own two primers form
        that product"""
        out = np.zeros(self.n_pairs, np.uint8)
        check(load().mpb_sites_own(self.h, lo, hi, ptr(out)))
        return out

    def close(self):
        if self.h:
            load().mpb_site_list_destroy(self.h)
            self.h = None


def words_of(n_rec: int) -> int:
    """32-bit words of one CoverMatrix row"""
    return max(4, -(-int(n_rec) // 128) * 4)


def cover_bytes(n_rows: int, n_rec: int) -> int:
    """device bytes of a CoverMatrix"""
    return (2 * int(n_rows) + 2) * words_of(n_rec) * 4


class Context:
    """one CUDA device + stream"""

    _shared = {}

    def __init__(self, device: int = 0, stream: int | None = None):
        lib = load()
        h = C.c_void_p()
        check(lib.mpb_ctx_create(device, C.byref(h)))
        self.h = h
        self.device = device
        self.is_shared = False
        if stream is not None:
            self.set_stream(stream)

    @classmethod
    def shared(cls, device: int = 0, stream: int | None = None) -> "Context":
        """the process-wide context of (device, stream): creating one costs a pinned allocation and a stream, which a
        caller that designs many alignments in a row (the Snakemake pipeline calls the CLI once per cluster, a server
        would not) should not pay per call.  close() leaves it open."""
        import threading
        key = (device, stream, threading.get_ident())
        ctx = cls._shared.get(key)
        if ctx is None or not ctx.h:
            ctx = cls(device, stream)
            ctx.is_shared = True
            cls._shared[key] = ctx
        return ctx

    def set_stream(self, stream: int):
        check(load().mpb_ctx_set_stream(self.h, C.c_void_p(stream)))

    def sync(self):
        check(load().mpb_ctx_sync(self.h))

    @property
    def launches(self) -> int:
        return load().mpb_ctx_launches(self.h)

    def profile(self, enable: bool = True):
        check(load().mpb_ctx_profile(self.h, int(enable)))

    def profile_read(self, kernel: str | None):
        """(total ms, launches, work units) of one kernel's event-timed launches; None clears the records"""
        ms, n, u = C.c_double(), C.c_int64(), C.c_double()
        check(load().mpb_ctx_profile_read(self.h, kernel.encode() if kernel else None, C.byref(ms), C.byref(n),
                                          C.byref(u)))
        return ms.value, n.value, u.value

    def primer_props(self, sets: np.ndarray, k: int, gc_lo: float, gc_hi: float, distance: int, consts3):
        """mpb_primer_props -> (tm_avg, gc, flags, deg, ndeg)"""
        sets = np.ascontiguousarray(sets, dtype=np.uint8)
        n = len(sets)
        cst = np.asarray(consts3, dtype=np.float64)
        tm = np.zeros(n, np.float64)
        gc = np.zeros(n, np.float64)
        flags = np.zeros(n, np.int32)
        deg = np.zeros(n, np.int32)
        ndeg = np.zeros(n, np.int32)
        if n:
            check(load().mpb_primer_props(self.h, ptr(sets), k, n, gc_lo, gc_hi, distance, ptr(cst), ptr(tm), ptr(gc),
                                          ptr(flags), ptr(deg), ptr(ndeg)))
        return tm, gc, flags, deg, ndeg

    def pair_cover(self, uf: np.ndarray, ur: np.ndarray, pf, pr) -> np.ndarray:
        """popcount(uf[pf] | ur[pr]) per pair (get_multiPrime.py:560-569 on bit vectors)"""
        uf = np.ascontiguousarray(uf, dtype=np.uint32)
        ur = np.ascontiguousarray(ur, dtype=np.uint32)
        pf = np.ascontiguousarray(pf, dtype=np.int32)
        pr = np.ascontiguousarray(pr, dtype=np.int32)
        out = np.zeros(len(pf), np.int32)
        if len(pf):
            check(load().mpb_pair_cover(self.h, ptr(uf), ptr(ur), uf.shape[0], uf.shape[1], ptr(pf), ptr(pr), len(pf),
                                        ptr(out)))
        return out

    def pair_cover3(self, bits, pf, pr) -> np.ndarray:
        """popcount(F[pf] | gap[pf] | R[pr] | gap[pr]) per pair on the scan's bit vectors bits[n, 3, words] (numpy or a
        DevBuf left in HBM by Hist.cscan)"""
        pf = np.ascontiguousarray(pf, dtype=np.int32)
        pr = np.ascontiguousarray(pr, dtype=np.int32)
        out = np.zeros(len(pf), np.int32)
        shape = bits.shape
        if isinstance(bits, np.ndarray):
            bits = np.ascontiguousarray(bits, dtype=np.uint32)
        if len(pf):
            check(load().mpb_pair_cover3(self.h, ptr(bits), shape[0], shape[2], ptr(pf), ptr(pr), len(pf), ptr(out)))
        return out

    def pool_search(self, w, n_pools: int, seed: int, r0: int, r1: int, iterations: int):
        """mpb_pool_search: restarts [r0, r1) of the pool search on the symmetric weights w[n, n] -> dict(cost int64[R],
        step int32[R], assign uint8[R, n]) per restart"""
        w = np.ascontiguousarray(w, dtype=np.uint8)
        n = w.shape[0] if w.ndim == 2 else 0
        nr = max(int(r1) - int(r0), 0)
        cost = np.zeros(nr, np.int64)
        step = np.zeros(nr, np.int32)
        assign = np.zeros((nr, max(n, 1)), np.uint8)
        if w.ndim != 2 or w.shape[0] != w.shape[1]:
            raise MpbError(-1, "w must be a square matrix (got shape %s)" % (w.shape,))
        check(load().mpb_pool_search(self.h, n, n_pools, ptr(w), int(seed) & 0xFFFFFFFFFFFFFFFF, r0, r1, iterations,
                                     ptr(cost), ptr(step), ptr(assign)))
        return dict(cost=cost, step=step, assign=assign[:, :n])

    def cover_gains(self, mat: CoverMatrix, cand) -> np.ndarray:
        """mpb_cover_gains -> int64[len(cand), 2]: new targets and new perfect targets of the listed rows"""
        cand = np.ascontiguousarray(cand, dtype=np.int32)
        out = np.zeros((len(cand), 2), np.int64)
        check(load().mpb_cover_gains(self.h, C.c_void_p(mat.amp), C.c_void_p(mat.perf), mat.n_rows, mat.words,
                                     C.c_void_p(mat.covered), C.c_void_p(mat.covered_perfect), ptr(cand), len(cand),
                                     ptr(out)))
        return out

    def cover_take(self, mat: CoverMatrix, row: int):
        """mpb_cover_take: the covered vectors |= row `row`"""
        check(load().mpb_cover_take(self.h, C.c_void_p(mat.amp), C.c_void_p(mat.perf), mat.n_rows, mat.words, int(row),
                                    C.c_void_p(mat.covered), C.c_void_p(mat.covered_perfect)))

    def close(self):
        if self.h and not self.is_shared:
            load().mpb_ctx_destroy(self.h)
            self.h = None

    # -- Tm -------------------------------------------------------------------------------------------
    def tm(self, seqs2bit: np.ndarray, consts3, want_hs: bool = False):
        n, k = seqs2bit.shape
        seqs2bit = np.ascontiguousarray(seqs2bit, dtype=np.uint8)
        cst = np.asarray(consts3, dtype=np.float64)
        tm = np.empty(n, np.float64)
        dh = np.empty(n, np.float64) if want_hs else None
        ds = np.empty(n, np.float64) if want_hs else None
        check(load().mpb_tm(self.h, ptr(seqs2bit), k, n, ptr(cst), ptr(tm), ptr(dh), ptr(ds)))
        return (tm, dh, ds) if want_hs else tm


class Msa:
    """an alignment resident in HBM (bit-planes)"""

    def __init__(self, ctx: Context, packed4, n_seq: int, n_col: int, row_bytes: int | None = None, lens=None):
        self.ctx = ctx
        self.n_seq, self.n_col = int(n_seq), int(n_col)
        row_bytes = row_bytes if row_bytes is not None else (n_col + 1) // 2
        if lens is not None:
            lens = np.ascontiguousarray(lens, dtype=np.int32)
        h = C.c_void_p()
        check(load().mpb_msa_upload(ctx.h, ptr(packed4), n_seq, n_col, row_bytes, ptr(lens), C.byref(h)))
        self.h = h

    def close(self):
        if self.h:
            load().mpb_msa_free(self.h)
            self.h = None

    def set_row0(self, row0: int):
        check(load().mpb_msa_set_row0(self.h, row0))

    def seq_attr(self):
        lead = np.empty(self.n_seq, np.int32)
        rstrip = np.empty(self.n_seq, np.int32)
        check(load().mpb_seq_attr(self.h, ptr(lead), ptr(rstrip)))
        return lead, rstrip

    def prefilter(self, k: int, v: int, win_pos):
        """(s0, s1) per window: see mpb_window_prefilter"""
        win_pos = np.ascontiguousarray(win_pos, dtype=np.int32)
        s0 = np.zeros(len(win_pos), np.float64)
        s1 = np.zeros(len(win_pos), np.float64)
        check(load().mpb_window_prefilter(self.h, k, v, ptr(win_pos), len(win_pos), ptr(s0), ptr(s1)))
        return s0, s1

    def seq_attr_hist(self):
        """histograms (value -> number of sequences) of the leading-gap count and of the length without trailing gaps"""
        lead = np.zeros(self.n_col + 1, np.int64)
        rstrip = np.zeros(self.n_col + 1, np.int64)
        check(load().mpb_seq_attr_hist(self.h, ptr(lead), ptr(rstrip)))
        return lead, rstrip

    def hist(self, k: int, v: int, win_pos, log2_cap: int = 0, empty: bool = False) -> "Hist":
        return Hist(self, k, v, win_pos, log2_cap, empty)

    def scan(self, k: int, v: int, fmask: int, rmask: int, cand_pos, cand_allow, bits_slot=None, counts_out=None,
             bits_out=None):
        """returns (counts[nc,3] int64, bits[nslots,3,words] uint32 or None)"""
        cand_pos = np.ascontiguousarray(cand_pos, dtype=np.int32)
        cand_allow = np.ascontiguousarray(cand_allow, dtype=np.uint32).reshape(-1, 4)
        nc = len(cand_pos)
        counts = counts_out if counts_out is not None else np.zeros((nc, 3), np.int64)
        bits = bits_out
        if bits_slot is not None:
            bits_slot = np.ascontiguousarray(bits_slot, dtype=np.int32)
            nslots = int(bits_slot.max()) + 1 if nc else 0
            words = (self.n_seq + 31) // 32
            if bits is None:
                bits = np.zeros((max(nslots, 0), 3, words), np.uint32)
        if nc:
            check(load().mpb_scan(self.h, k, v, fmask, rmask, ptr(cand_pos), ptr(cand_allow), nc, ptr(counts),
                                  ptr(bits_slot), ptr(bits)))
        return counts, bits

    def pattern_hits(self, allow, lens, max_hits: int = 1 << 20):
        """mpb_pattern_hits: every exact occurrence of the degenerate patterns -> (pattern, sequence, position) arrays
        sorted by (pattern, sequence, position)"""
        allow = np.ascontiguousarray(allow, dtype=np.uint32).reshape(-1, 4)
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        while True:
            hp, hr, hx = (np.empty(max_hits, np.int32) for _ in range(3))
            n = C.c_int64()
            check(load().mpb_pattern_hits(self.h, len(lens), ptr(allow), ptr(lens), max_hits, ptr(hp), ptr(hr), ptr(hx),
                                          C.byref(n)))
            if n.value <= max_hits:
                break
            max_hits = int(n.value) + 16
        n = n.value
        order = np.lexsort((hx[:n], hr[:n], hp[:n]))
        return hp[:n][order], hr[:n][order], hx[:n][order]

    def pattern_sites(self, allow, lens, strict, v: int, max_hits: int = 1 << 20):
        """mpb_pattern_sites: every site of the degenerate patterns with at most v mismatches and none at a strict
        position -> (pattern, sequence, position, mismatches) arrays sorted by (pattern, sequence, position)"""
        allow = np.ascontiguousarray(allow, dtype=np.uint32).reshape(-1, 4)
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        strict = np.ascontiguousarray(strict, dtype=np.uint32)
        while True:
            hp, hr, hx, hm = (np.empty(max_hits, np.int32) for _ in range(4))
            n = C.c_int64()
            check(load().mpb_pattern_sites(self.h, len(lens), ptr(allow), ptr(lens), ptr(strict), v, max_hits, ptr(hp),
                                           ptr(hr), ptr(hx), ptr(hm), C.byref(n)))
            if n.value <= max_hits:
                break
            max_hits = int(n.value) + 16
        n = n.value
        order = np.lexsort((hx[:n], hr[:n], hp[:n]))
        return hp[:n][order], hr[:n][order], hx[:n][order], hm[:n][order]

    def pattern_products(self, allow, lens, strict, v: int, pat_primer, pat_side, n_primer: int, stride: int, rec_off,
                         rec_len, lo: int, hi: int, listed, max_rows: int, chunk: int = 0):
        """mpb_pattern_products: products of every (left primer i, right primer j) combination in the records, joined on
        the device -> dict(comb int64[n_primer, n_primer, 3] (products, targets, perfect targets), union int64[2]
        (targets and perfect targets over the combinations flagged in listed[n_primer, n_primer]), rows int64[n, 8]
        (the first max_rows listed groups: record, i, j, start, length, left / right mismatches, products), n_listed,
        stats int64[4] (search hits, left sites, right sites, groups))"""
        allow = np.ascontiguousarray(allow, dtype=np.uint32).reshape(-1, 4)
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        strict = np.ascontiguousarray(strict, dtype=np.uint32)
        pat_primer = np.ascontiguousarray(pat_primer, dtype=np.int32)
        pat_side = np.ascontiguousarray(pat_side, dtype=np.int32)
        rec_off = np.ascontiguousarray(rec_off, dtype=np.int64)
        rec_len = np.ascontiguousarray(rec_len, dtype=np.int64)
        listed = np.ascontiguousarray(listed, dtype=np.uint8).reshape(n_primer, n_primer)
        comb = np.zeros((n_primer, n_primer, 3), np.int64)
        uni = np.zeros(2, np.int64)
        rows = np.zeros((max(max_rows, 1), 8), np.int64)
        stats = np.zeros(4, np.int64)
        n = C.c_int64()
        check(load().mpb_pattern_products(self.h, len(lens), ptr(allow), ptr(lens), ptr(strict), v, ptr(pat_primer),
                                          ptr(pat_side), n_primer, stride, len(rec_off), ptr(rec_off), ptr(rec_len), lo,
                                          hi, ptr(listed), chunk, max_rows, ptr(comb), ptr(uni), ptr(rows), C.byref(n),
                                          ptr(stats)))
        return dict(comb=comb, union=uni, rows=rows[:min(n.value, max_rows)], n_listed=n.value, stats=stats)

    def pattern_cover(self, allow, lens, strict, v: int, stride: int, rec_off, rec_len, lo: int, hi: int,
                      mat: CoverMatrix, row0: int = 0, max_sites: int = 0) -> np.ndarray:
        """mpb_pattern_cover: the amp / perf bits of the pairs row0, row0 + 1, ... of mat (four patterns each, Panel
        order) over the records -> stats int64[3] (search hits, left sites, right sites).  max_sites: the search's
        first capacity (0: the library's default); a search that finds more sites runs a second time."""
        allow = np.ascontiguousarray(allow, dtype=np.uint32).reshape(-1, 4)
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        strict = np.ascontiguousarray(strict, dtype=np.uint32)
        rec_off = np.ascontiguousarray(rec_off, dtype=np.int64)
        rec_len = np.ascontiguousarray(rec_len, dtype=np.int64)
        if len(rec_off) != mat.n_rec or not 0 <= row0 <= row0 + len(lens) // 4 <= mat.n_rows:
            raise MpbError(-1, "pairs %d.. / %d records do not fit the %d x %d matrix" % (row0, len(rec_off), mat.n_rows,
                                                                                          mat.n_rec))
        stats = np.zeros(3, np.int64)
        off = row0 * mat.words * 4
        check(load().mpb_pattern_cover(self.h, len(lens), ptr(allow), ptr(lens), ptr(strict), v, stride, len(rec_off),
                                       ptr(rec_off), ptr(rec_len), lo, hi, mat.words, C.c_void_p(mat.amp + off),
                                       C.c_void_p(mat.perf + off), int(max_sites), ptr(stats)))
        return stats

    def pattern_cover_keep(self, allow, lens, strict, v: int, stride: int, rec_off, rec_len, lo: int, hi: int,
                           mat: CoverMatrix | None, row0: int, max_sites: int, sites: "SiteList") -> np.ndarray:
        """mpb_pattern_cover_keep: pattern_cover (mat None: no matrix, search only) that also appends its filtered
        sites to `sites` as the patterns 4 * row0, ... of the list -> stats int64[3]"""
        allow = np.ascontiguousarray(allow, dtype=np.uint32).reshape(-1, 4)
        lens = np.ascontiguousarray(lens, dtype=np.int32)
        strict = np.ascontiguousarray(strict, dtype=np.uint32)
        rec_off = np.ascontiguousarray(rec_off, dtype=np.int64)
        rec_len = np.ascontiguousarray(rec_len, dtype=np.int64)
        amp = perf = None
        words = 0
        if mat is not None:
            if len(rec_off) != mat.n_rec or not 0 <= row0 <= row0 + len(lens) // 4 <= mat.n_rows:
                raise MpbError(-1, "pairs %d.. / %d records do not fit the %d x %d matrix" % (
                    row0, len(rec_off), mat.n_rows, mat.n_rec))
            off = row0 * mat.words * 4
            amp, perf, words = C.c_void_p(mat.amp + off), C.c_void_p(mat.perf + off), mat.words
        stats = np.zeros(3, np.int64)
        check(load().mpb_pattern_cover_keep(self.h, len(lens), ptr(allow), ptr(lens), ptr(strict), v, stride,
                                            len(rec_off), ptr(rec_off), ptr(rec_len), lo, hi, words, amp, perf,
                                            int(max_sites), ptr(stats), sites.h, 4 * int(row0)))
        return stats

    def seqkeys(self, k: int, win_pos) -> np.ndarray:
        win_pos = np.ascontiguousarray(win_pos, dtype=np.int32)
        out = np.empty((len(win_pos), self.n_seq), np.uint64)
        check(load().mpb_seqkeys(self.h, k, ptr(win_pos), len(win_pos), ptr(out)))
        return out


class Hist:
    """per-window haplotype tables of one window batch"""

    def __init__(self, msa: Msa, k: int, v: int, win_pos, log2_cap: int = 0, empty: bool = False):
        self.msa = msa
        self.k, self.v = k, v
        self.win_pos = np.ascontiguousarray(win_pos, dtype=np.int32)
        self.nw = len(self.win_pos)
        self.h = None
        cap = log2_cap
        if empty:                       # owner tables of a sequence-sharded run: filled through merge() only
            h = C.c_void_p()
            check(load().mpb_hist_create_empty(msa.h, k, v, ptr(self.win_pos), self.nw, cap, C.byref(h)))
            self.h = h
            self.log2_cap = cap
            return
        while True:
            h = C.c_void_p()
            rc = load().mpb_hist_build(msa.h, k, v, ptr(self.win_pos), self.nw, cap, C.byref(h))
            if rc == -4:  # MPB_EOVERFLOW: IUPAC expansions outgrew the table, double it
                if cap == 0:
                    cap = max(6, int(np.ceil(np.log2(2 * msa.n_seq + 64))))
                cap += 1
                continue
            check(rc)
            self.h = h
            self.log2_cap = cap
            break

    def close(self):
        if self.h:
            load().mpb_hist_free(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def summary(self):
        """mpb_hist_summary: stats() and tensors() of every window in one pass over the occupied slots"""
        nw, k = self.nw, self.k
        out = dict(gap_n=np.empty(nw, np.int64), ent=np.empty((nw, 4), np.float64), nuniq=np.empty((nw, 3), np.int64),
                   mm_key=np.empty(nw, np.uint64), mm_cnt=np.empty(nw, np.int64), mm_first=np.empty(nw, np.uint64),
                   n_iupac_gap=np.empty(nw, np.int64), freq=np.empty((nw, 4, k), np.int64),
                   nn=np.empty((nw, k - 1, 4, 4), np.int64))
        check(load().mpb_hist_summary(self.h, ptr(out["gap_n"]), ptr(out["ent"]), ptr(out["nuniq"]), ptr(out["mm_key"]),
                                      ptr(out["mm_cnt"]), ptr(out["mm_first"]), ptr(out["n_iupac_gap"]),
                                      ptr(out["freq"]), ptr(out["nn"])))
        return out

    def add_counts(self, gap_n, n_iupac_gap):
        gap_n = np.ascontiguousarray(gap_n, dtype=np.int64)
        n_iupac_gap = np.ascontiguousarray(n_iupac_gap, dtype=np.int64)
        check(load().mpb_hist_add_counts(self.h, ptr(gap_n), ptr(n_iupac_gap)))

    def cscan(self, fmask: int, rmask: int, cands: np.ndarray, bits_slot=None, counts_out=None, bits_out=None):
        """mpb_cscan: column scan of CAND_DTYPE candidates -> (counts[nc,4] int64, bits[nslots,3,words] uint32 or None)"""
        cands = np.ascontiguousarray(cands, dtype=CAND_DTYPE)
        nc = len(cands)
        counts = counts_out if counts_out is not None else np.zeros((nc, 4), np.int64)
        bits = bits_out
        if bits_slot is not None:
            bits_slot = np.ascontiguousarray(bits_slot, dtype=np.int32)
            nslots = int(bits_slot.max()) + 1 if nc else 0
            if bits is None:
                bits = np.zeros((max(nslots, 0), 3, (self.msa.n_seq + 31) // 32), np.uint32)
            elif bits == "device":      # stay in HBM (pair coverage reads them there)
                bits = DevBuf(self.msa.ctx, (max(nslots, 1), 3, (self.msa.n_seq + 31) // 32), np.uint32)
        if nc:
            check(load().mpb_cscan(self.h, fmask, rmask, ptr(cands), nc, ptr(counts), ptr(bits_slot), ptr(bits)))
        return counts, bits

    def walk(self, dnum, degeneracy, fmask, rmask, win_idx, cover_number, mm_key, freq=None, nn=None, comm=None,
             want_trace=True, lag=2, peer=None):
        """the device-resident refinement walk of the windows win_idx (indices into this batch) -> walk() outputs.
        comm (sequence shards): the count vector is summed over the ranks between scan and advance — inside the round's
        kernel chain through `peer` (NVLink peer memory), else by the communicator's all-reduce, one host call per round."""
        with WalkDev(self, dnum, degeneracy, fmask, rmask, win_idx, cover_number, mm_key, freq, nn) as w:
            if comm is None or comm.world == 1 or (peer is not None and w.set_peer(peer)):
                w.run(lag)
            else:
                on_gpu = getattr(comm, "on_gpu", False)
                counts_t = w.counts_tensor(comm) if on_gpu else None
                r = 0
                while True:
                    w.advance()
                    if r >= lag and w.wait(r - lag) == 0:       # identical on every rank: same counts, same rounds
                        break
                    w.scan()
                    if on_gpu:
                        comm.allreduce_dev_inplace(counts_t)    # NCCL over NVLink, on the context's stream
                    else:                                       # host communicator (gloo): through host memory
                        w.set_counts(comm.allreduce_sum(w.get_counts()))
                    r += 1
            return w.finish(want_trace)

    def stats(self):
        nw = self.nw
        out = dict(gap_n=np.empty(nw, np.int64), ent=np.empty((nw, 4), np.float64), nuniq=np.empty((nw, 3), np.int64),
                   mm_key=np.empty(nw, np.uint64), mm_cnt=np.empty(nw, np.int64), mm_first=np.empty(nw, np.uint64),
                   n_iupac_gap=np.empty(nw, np.int64))
        check(load().mpb_hist_stats(self.h, ptr(out["gap_n"]), ptr(out["ent"]), ptr(out["nuniq"]), ptr(out["mm_key"]),
                                    ptr(out["mm_cnt"]), ptr(out["mm_first"]), ptr(out["n_iupac_gap"])))
        return out

    def counts(self):
        """(gap rows, gap rows holding IUPAC cells, distinct entries) per window, from the build counters"""
        out = [np.zeros(self.nw, np.int64) for _ in range(3)]
        check(load().mpb_hist_counts(self.h, ptr(out[0]), ptr(out[1]), ptr(out[2])))
        return out

    def tensors(self, sel):
        sel = np.ascontiguousarray(sel, dtype=np.uint8)
        freq = np.empty((self.nw, 4, self.k), np.int64)
        nn = np.empty((self.nw, self.k - 1, 4, 4), np.int64)
        check(load().mpb_hist_tensors(self.h, ptr(sel), ptr(freq), ptr(nn)))
        return freq, nn

    def dump(self, w: int, max_n: int):
        keys = np.empty(max_n, np.uint64)
        cnt = np.empty(max_n, np.uint32)
        first = np.empty(max_n, np.uint64)
        n = C.c_int64()
        check(load().mpb_hist_dump(self.h, w, max_n, ptr(keys), ptr(cnt), ptr(first), C.byref(n)))
        n = min(n.value, max_n)
        order = np.argsort(first[:n], kind="stable")
        return keys[:n][order], cnt[:n][order], first[:n][order]

    def export(self, sel, counts):
        """entries of the selected windows; counts[w] = entries of window w -> (win_off, keys, cnt, first)"""
        sel = np.ascontiguousarray(sel, dtype=np.uint8)
        off = np.zeros(self.nw + 1, np.int64)
        off[1:] = np.cumsum(np.where(sel != 0, counts, 0))
        total = int(off[-1])
        keys = np.empty(total, np.uint64)
        cnt = np.empty(total, np.uint32)
        first = np.empty(total, np.uint64)
        if total:
            check(load().mpb_hist_export(self.h, ptr(sel), ptr(off), ptr(keys), ptr(cnt), ptr(first)))
        return off, keys, cnt, first

    def merge(self, win_off, keys, cnt, first):
        win_off = np.ascontiguousarray(win_off, dtype=np.int64)
        if win_off[-1] > 0:
            if isinstance(keys, np.ndarray):
                keys = np.ascontiguousarray(keys, dtype=np.uint64)
                cnt = np.ascontiguousarray(cnt, dtype=np.uint32)
                first = np.ascontiguousarray(first, dtype=np.uint64)
            check(load().mpb_hist_merge(self.h, ptr(win_off), ptr(keys), ptr(cnt), ptr(first)))

    def export_at(self, order, counts, comm=None):
        """entries of the windows `order` (batch indices, in this order), counts[i] of window order[i] -> (keys, cnt,
        first) compact arrays; device tensors allocated through comm when it is on the GPU, numpy otherwise"""
        order = np.ascontiguousarray(order, dtype=np.int32)
        room = np.ascontiguousarray(counts, dtype=np.int64)
        start = np.zeros(len(order), np.int64)
        start[1:] = np.cumsum(room)[:-1]
        total = int(room.sum())
        if comm is not None:
            keys, cnt, first = comm.empty_dev(total, np.uint64), comm.empty_dev(total, np.uint32), comm.empty_dev(total, np.uint64)
        else:
            keys, cnt, first = np.empty(total, np.uint64), np.empty(total, np.uint32), np.empty(total, np.uint64)
        if total:
            check(load().mpb_hist_export_at(self.h, len(order), ptr(order), ptr(start), ptr(room), total, ptr(keys),
                                            ptr(cnt), ptr(first)))
        return keys, cnt, first

    def merge_segments(self, seg_off, keys, cnt, first):
        """merge() for m * nw segments: segment s belongs to window s % nw (keys / cnt / first: numpy or device tensors)"""
        seg_off = np.ascontiguousarray(seg_off, dtype=np.int64)
        if seg_off[-1] > 0:
            if isinstance(keys, np.ndarray):
                keys = np.ascontiguousarray(keys, dtype=np.uint64)
                cnt = np.ascontiguousarray(cnt, dtype=np.uint32)
                first = np.ascontiguousarray(first, dtype=np.uint64)
            check(load().mpb_hist_merge_segments(self.h, len(seg_off) - 1, ptr(seg_off), ptr(keys), ptr(cnt), ptr(first)))

    def export_dev(self, sel, counts, comm):
        """export() into device tensors allocated through the communicator -> (win_off, keys, cnt, first)"""
        sel = np.ascontiguousarray(sel, dtype=np.uint8)
        off = np.zeros(self.nw + 1, np.int64)
        off[1:] = np.cumsum(np.where(sel != 0, counts, 0))
        total = int(off[-1])
        keys = comm.empty_dev(total, np.uint64)
        cnt = comm.empty_dev(total, np.uint32)
        first = comm.empty_dev(total, np.uint64)
        if total:
            check(load().mpb_hist_export(self.h, ptr(sel), ptr(off), ptr(keys), ptr(cnt), ptr(first)))
        return off, keys, cnt, first

    def match(self, q_win, q_allow):
        q_win = np.ascontiguousarray(q_win, dtype=np.int32)
        q_allow = np.ascontiguousarray(q_allow, dtype=np.uint32).reshape(-1, 4)
        out = np.zeros(len(q_win), np.int64)
        if len(q_win):
            check(load().mpb_hist_match(self.h, ptr(q_win), ptr(q_allow), len(q_win), ptr(out)))
        return out

    def exceptions(self):
        n = C.c_int64()
        check(load().mpb_hist_exceptions(self.h, 0, None, None, C.byref(n)))
        w = np.empty(n.value, np.int32)
        s = np.empty(n.value, np.int32)
        if n.value:
            check(load().mpb_hist_exceptions(self.h, n.value, ptr(w), ptr(s), C.byref(n)))
        return w, s


PEER_HANDLE_BYTES = 128
PEER_MAX_WORLD = 8


class Peer:
    """mpb_peer_*: one rank's member of a peer-memory group (one rank per GPU, NVLink): the walk's count vector is summed
    over the ranks by one small kernel per round instead of a collective-library call."""

    def __init__(self, ctx: Context, rank: int, world: int, cap_elems: int = 1 << 18):
        self.ctx, self.rank, self.world, self.cap = ctx, rank, world, int(cap_elems)
        h = C.c_void_p()
        check(load().mpb_peer_create(ctx.h, rank, world, self.cap, C.byref(h)))
        self.h = h

    def handle(self) -> np.ndarray:
        out = np.zeros(PEER_HANDLE_BYTES // 8, np.int64)
        check(load().mpb_peer_handle(self.h, ptr(out)))
        return out

    def connect(self, handles):
        handles = np.ascontiguousarray(handles, dtype=np.int64)
        assert handles.shape == (self.world, PEER_HANDLE_BYTES // 8)
        check(load().mpb_peer_connect(self.h, ptr(handles)))

    @classmethod
    def of(cls, ctx: Context, comm, cap_elems: int = 1 << 18):
        """The member of this process in the group of `comm` (cached on the context: opening IPC handles costs
        milliseconds), or None when the group cannot be used — a rank failed to create or open a buffer, or the trial
        all-reduce did not give the expected sum.  Every step is agreed on by all ranks through `comm`, so either all of
        them use peer memory or none does (the walk then all-reduces through the communicator)."""
        cache = ctx.__dict__.setdefault("_peers", {})
        key = (getattr(comm, "peer_key", None), comm.rank, comm.world)
        if key in cache:
            return cache[key]
        peer, words = None, PEER_HANDLE_BYTES // 8
        mine = np.zeros(words + 1, np.int64)
        try:
            peer = cls(ctx, comm.rank, comm.world, cap_elems)
            mine[:words] = peer.handle()
            mine[words] = 1
        except MpbError:
            peer = None
        everyone = comm.allgather_fixed(mine)
        ok = bool(everyone[:, words].all())
        if ok:
            try:
                peer.connect(everyone[:, :words])
            except MpbError:
                ok = False
        ok = int(comm.allreduce_sum(np.array([1 if ok else 0], np.int64))[0]) == comm.world
        if ok:                               # (the barrier inside the all-reduce: every rank has opened every buffer)
            trial = DevBuf(ctx, (8,), np.int64)
            try:
                want = np.arange(8, dtype=np.int64) * comm.world + comm.world * (comm.world + 1) // 2
                check(load().mpb_ctx_memcpy(ctx.h, C.c_void_p(trial.p), ptr(np.arange(8, dtype=np.int64) + comm.rank + 1), 64))
                peer.allreduce(trial.p, 8)
                ok = bool((trial.to_host() == want).all())
            except MpbError:
                ok = False
            finally:
                trial.close()
            ok = int(comm.allreduce_sum(np.array([1 if ok else 0], np.int64))[0]) == comm.world
        if not ok and peer is not None:
            peer.close()
            peer = None
        cache[key] = peer
        return peer

    def allreduce(self, dev_ptr: int, n: int, phases: int = 3):
        check(load().mpb_peer_allreduce_phases(self.h, C.c_void_p(dev_ptr), n, phases))

    def close(self):
        if self.h:
            load().mpb_peer_free(self.h)
            self.h = None


class WalkDev:
    """mpb_walk_dev_*: tracks resident in HBM, rounds chained on the context's stream"""

    def __init__(self, hist: Hist, dnum, degeneracy, fmask, rmask, win_idx, cover_number, mm_key, freq=None, nn=None):
        self.hist = hist
        self.n = len(win_idx)
        win_idx = np.ascontiguousarray(win_idx, dtype=np.int32)
        cover_number = np.ascontiguousarray(cover_number, dtype=np.int64)
        mm_key = np.ascontiguousarray(mm_key, dtype=np.uint64)
        if freq is not None and isinstance(freq, np.ndarray):
            freq = np.ascontiguousarray(freq, dtype=np.int64)
            nn = np.ascontiguousarray(nn, dtype=np.int64)
        h = C.c_void_p()
        check(load().mpb_walk_dev_begin(hist.h, dnum, degeneracy, fmask, rmask, self.n, ptr(win_idx), ptr(cover_number),
                                        ptr(mm_key), ptr(freq), ptr(nn), C.byref(h)))
        self.h = h
        self._inputs = (win_idx, cover_number, mm_key, freq, nn)     # alive until the walk is done

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def close(self):
        if self.h:
            load().mpb_walk_dev_free(self.h)
            self.h = None

    def set_peer(self, peer) -> bool:
        """all-reduce the counts through the peer group; False when a round could exceed the group's capacity"""
        if 2 * self.n * (self.hist.k - 1) * 4 > peer.cap:
            return False
        check(load().mpb_walk_dev_set_peer(self.h, peer.h))
        return True

    def advance(self):
        check(load().mpb_walk_dev_advance(self.h))

    def scan(self):
        check(load().mpb_walk_dev_scan(self.h))

    def wait(self, rnd: int) -> int:
        live = C.c_int64()
        check(load().mpb_walk_dev_wait(self.h, rnd, C.byref(live)))
        return live.value

    def run(self, lag: int = 2) -> int:
        rounds = C.c_int64()
        check(load().mpb_walk_dev_run(self.h, lag, C.byref(rounds)))
        return rounds.value

    def counts_tensor(self, comm):
        """the device count vector as a tensor of the communicator's framework (no copy)"""
        p, n = C.c_void_p(), C.c_int64()
        check(load().mpb_walk_dev_counts(self.h, C.byref(p), C.byref(n)))
        return comm.wrap_dev(p.value, n.value)

    def _counts_ptr(self):
        p, n = C.c_void_p(), C.c_int64()
        check(load().mpb_walk_dev_counts(self.h, C.byref(p), C.byref(n)))
        return p, n.value

    def get_counts(self) -> np.ndarray:
        p, n = self._counts_ptr()
        out = np.empty(n, np.int64)
        check(load().mpb_ctx_memcpy(self.hist.msa.ctx.h, ptr(out), p, n * 8))
        return out

    def set_counts(self, arr: np.ndarray):
        p, n = self._counts_ptr()
        arr = np.ascontiguousarray(arr, dtype=np.int64)
        assert len(arr) == n
        check(load().mpb_ctx_memcpy(self.hist.msa.ctx.h, p, ptr(arr), n * 8))

    def finish(self, want_trace=True):
        n = self.n
        res = _walk_outputs(n)
        cap = n * 2 * 48 if want_trace else 0
        trace = np.zeros((cap, 32), np.uint8) if want_trace else None
        off = np.zeros(n + 1, np.int64)
        check(load().mpb_walk_dev_finish(self.h, ptr(res["sets"]), ptr(res["counts"]), ptr(res["seeds"]),
                                         ptr(res["seed_cover"]), ptr(res["ntracks"]), cap, ptr(trace), ptr(off),
                                         ptr(res["stats"])))
        res.update(trace=trace, trace_off=off)
        return res


class Dimer:
    """expansions + 3' end tables of a primer list on the device; pair queries (include/mpb200.h mpb_dimer_*)"""

    def __init__(self, ctx: Context, sets_list, min_end: int, max_end: int, init_both: bool, loss_table: np.ndarray,
                 dg_consts):
        n = len(sets_list)
        sets = np.zeros((n, 32), np.uint8)
        lens = np.zeros(n, np.int32)
        for i, s in enumerate(sets_list):
            sets[i, :len(s)] = s
            lens[i] = len(s)
        self.n = n
        self.lens = lens
        cst = np.ascontiguousarray(dg_consts, dtype=np.float64)
        tab = np.ascontiguousarray(loss_table, dtype=np.uint8)
        assert tab.shape == (33, 33, 33) and cst.shape == (24,)
        h = C.c_void_p()
        check(load().mpb_dimer_prepare(ctx.h, ptr(sets), ptr(lens), n, min_end, max_end, int(init_both), ptr(tab),
                                       ptr(cst), C.byref(h)))
        self.h = h
        self.off_p = np.zeros(n + 1, np.int64)
        self.off_e = np.zeros(n + 1, np.int64)
        check(load().mpb_dimer_counts(self.h, ptr(self.off_p), ptr(self.off_e)))

    def pairs(self, pi, pj):
        """first hit per pair: (order index or -1, d2)"""
        pi = np.ascontiguousarray(pi, dtype=np.int32)
        pj = np.ascontiguousarray(pj, dtype=np.int32)
        hit = np.full(len(pi), -1, np.int64)
        d2 = np.full(len(pi), -1, np.int32)
        if len(pi):
            check(load().mpb_dimer_pairs(self.h, ptr(pi), ptr(pj), len(pi), ptr(hit), ptr(d2)))
        return hit, d2

    def grid(self, row0: int, row1: int, max_hits: int = 1 << 22):
        """dimer pairs (i in [row0,row1), j >= i) -> (i, j, order index, d2, pairs tested after the prefilter)"""
        hi = np.empty(max_hits, np.int32)
        hj = np.empty(max_hits, np.int32)
        ho = np.empty(max_hits, np.int64)
        hd = np.empty(max_hits, np.int32)
        n, nt = C.c_int64(), C.c_int64()
        check(load().mpb_dimer_grid(self.h, row0, row1, max_hits, ptr(hi), ptr(hj), ptr(ho), ptr(hd), C.byref(n),
                                    C.byref(nt)))
        n = n.value
        return hi[:n], hj[:n], ho[:n], hd[:n], nt.value

    def close(self):
        if self.h:
            load().mpb_dimer_free(self.h)
            self.h = None
