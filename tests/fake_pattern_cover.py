"""The CPU double of mpb_pattern_cover, mpb_cover_gains and mpb_cover_take, on top of tests/fake_pattern_sites.py (its
search) and tests/fake_device.py (its Context and Dimer).

TEST INFRASTRUCTURE ONLY: pass this module as the backend of multiprime_b200.primer_select to run the tool's host logic
(blocks, sharding, the greedy, writing) without a GPU; tests/test_gpu_pattern_cover.py pins the real entry points to
this double and to primer_coverage.amplicons."""
from __future__ import annotations

import numpy as np

from multiprime_b200._lib import MpbError, words_of
from tests.fake_device import Context as _Context
from tests.fake_device import Dimer  # noqa: F401  (the backend's Dimer)
from tests.fake_pattern_sites import Msa as _Msa


def _bits_for(n: int) -> int:
    b = 1
    while (1 << b) < n:
        b += 1
    return b


class CoverMatrix:
    """host arrays in the layout of multiprime_b200._lib.CoverMatrix"""

    def __init__(self, ctx, n_rows: int, n_rec: int):
        self.ctx, self.n_rows, self.n_rec = ctx, int(n_rows), int(n_rec)
        self.words = words_of(n_rec)
        self.buf = np.zeros((2 * self.n_rows + 2, self.words), np.uint32)

    def to_host(self):
        n = self.n_rows
        return self.buf[:n].copy(), self.buf[n:2 * n].copy(), self.buf[2 * n].copy(), self.buf[2 * n + 1].copy()

    def close(self):
        pass


def cover_rows(sites, plen, n_pairs, stride, rec_off, rec_len, lo, hi):
    """(pair, record, perfect) of every (pair, record) with an amplicon, from the row sites (pattern, row, x, mismatches)
    as mpb_pattern_cover states the rule"""
    hp, hr, hx, hm = (np.asarray(a, np.int64) for a in sites)
    g = hr * stride + hx
    rec = np.searchsorted(rec_off, g, side="right") - 1
    keep = (hx < stride) & (rec >= 0)
    rec = np.maximum(rec, 0)
    keep &= g + plen[hp] <= rec_off[rec] + rec_len[rec]
    hp, rec, g, hm = hp[keep], rec[keep], g[keep], hm[keep]
    out = set()
    perfect = set()
    for p in range(0, 4 * n_pairs, 2):
        lsel, rsel = hp == p, hp == p + 1
        ry = np.sort(g[rsel])
        ry0 = np.sort(g[rsel & (hm == 0)])
        ll, rl = int(plen[p]), int(plen[p + 1])
        for x, r, m in zip(g[lsel].tolist(), rec[lsel].tolist(), hm[lsel].tolist()):
            end = int(rec_off[r] + rec_len[r])
            ylo, yhi = x + max(ll, lo - rl), min(x + hi - rl, end - rl)
            if ylo > yhi:
                continue
            if np.searchsorted(ry, yhi, side="right") > np.searchsorted(ry, ylo):
                out.add((p // 4, r))
                if m == 0 and np.searchsorted(ry0, yhi, side="right") > np.searchsorted(ry0, ylo):
                    perfect.add((p // 4, r))
    return sorted((q, r, (q, r) in perfect) for q, r in out)


class Msa(_Msa):
    def pattern_cover(self, allow, lens, strict, v, stride, rec_off, rec_len, lo, hi, mat, row0=0, max_sites=0):
        lens = np.asarray(lens, np.int64)
        n_pat = len(lens)
        rec_off = np.asarray(rec_off, np.int64)
        rec_len = np.asarray(rec_len, np.int64)
        if n_pat < 4 or n_pat % 4:
            raise MpbError(-1, "%d patterns: four per pair are needed" % n_pat)
        if v < 0:
            raise MpbError(-1, "negative mismatch bound %d" % v)
        if not 0 < lo <= hi:
            raise MpbError(-1, "product lengths %d..%d: need 0 < lo <= hi" % (lo, hi))
        if len(rec_off) != mat.n_rec or not 0 <= row0 <= row0 + n_pat // 4 <= mat.n_rows:
            raise MpbError(-1, "pairs / records do not fit the matrix")
        if not 0 <= max_sites <= 1 << 31:
            raise MpbError(-1, "max_sites %d outside 0..2^31" % max_sites)
        if len(rec_off) and rec_off[-1] + rec_len[-1] > len(self.rows) * stride:
            raise MpbError(-1, "the last record ends past the stream columns of the rows")
        if _bits_for(n_pat) + _bits_for(len(self.rows) * stride) + 4 > 64:
            raise MpbError(-1, "the site key needs more than 64 bits")
        stats = np.zeros(3, np.int64)
        if not len(rec_off):
            return stats
        sites = self.pattern_sites(allow, lens, strict, v)
        stats[0] = len(sites[0])
        hp, hr, hx = (np.asarray(a, np.int64) for a in sites[:3])
        g = hr * stride + hx
        rec = np.searchsorted(rec_off, g, side="right") - 1
        keep = (hx < stride) & (rec >= 0)
        keep &= g + lens[hp] <= rec_off[np.maximum(rec, 0)] + rec_len[np.maximum(rec, 0)]
        stats[1], stats[2] = (keep & (hp % 2 == 0)).sum(), (keep & (hp % 2 == 1)).sum()
        n = mat.n_rows
        for q, r, perf in cover_rows(sites, lens, n_pat // 4, stride, rec_off, rec_len, lo, hi):
            mat.buf[row0 + q, r >> 5] |= np.uint32(1 << (r & 31))
            if perf:
                mat.buf[n + row0 + q, r >> 5] |= np.uint32(1 << (r & 31))
        return stats


def _popcount(a):
    return np.unpackbits(np.ascontiguousarray(a).view(np.uint8), axis=-1).sum(axis=-1).astype(np.int64)


class Context(_Context):
    def cover_gains(self, mat, cand):
        cand = np.asarray(cand, np.int64)
        if len(cand) and (cand.min() < 0 or cand.max() >= mat.n_rows):
            raise MpbError(-1, "candidate row outside 0..%d" % (mat.n_rows - 1))
        n = mat.n_rows
        amp, perf = mat.buf[cand], mat.buf[n + cand]
        cov, covp = mat.buf[2 * n], mat.buf[2 * n + 1]
        out = np.zeros((len(cand), 2), np.int64)
        if len(cand):
            out[:, 0] = _popcount(amp & ~cov)
            out[:, 1] = _popcount(perf & ~covp)
        return out

    def cover_take(self, mat, row):
        n = mat.n_rows
        if not 0 <= row < n:
            raise MpbError(-1, "row %d outside 0..%d" % (row, n - 1))
        mat.buf[2 * n] |= mat.buf[row]
        mat.buf[2 * n + 1] |= mat.buf[n + row]
