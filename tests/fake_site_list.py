"""The CPU double of mpb_site_list (create, mpb_pattern_cover_keep, seal, keys), mpb_sites_cross and mpb_sites_own, on
top of tests/fake_pattern_cover.py (its search, filter, matrix, Context and Dimer).

TEST INFRASTRUCTURE ONLY: pass this module as the backend of multiprime_b200.primer_select to run the tool's --cross /
--background host logic without a GPU; tests/test_gpu_site_list.py pins the real entry points to this double."""
from __future__ import annotations

import numpy as np

from multiprime_b200._lib import MpbError
from tests.fake_pattern_cover import Context, CoverMatrix, Dimer, _bits_for  # noqa: F401  (the backend's classes)
from tests.fake_pattern_cover import Msa as _Msa

PRIMER_OF = np.array([0, 1, 1, 0], np.int64)           # pattern % 4 -> 0 = F, 1 = R


class SiteList:
    """host keys in the layout of multiprime_b200._lib.SiteList"""

    def __init__(self, ctx, lens, n_pos: int, rec_off, rec_len):
        self.lens = np.asarray(lens, np.int64)
        self.rec_off = np.asarray(rec_off, np.int64)
        self.rec_len = np.asarray(rec_len, np.int64)
        n_pat = len(self.lens)
        if n_pat < 4 or n_pat % 4:
            raise MpbError(-1, "%d patterns: four per pair are needed" % n_pat)
        self.pat_bits, self.pos_bits = _bits_for(n_pat), _bits_for(int(n_pos))
        if self.pat_bits + self.pos_bits + 4 > 64:
            raise MpbError(-1, "the site key needs more than 64 bits")
        if len(self.rec_off) and self.rec_off[-1] + self.rec_len[-1] > n_pos:
            raise MpbError(-1, "a record ends past the stream columns")
        self.n_pairs = n_pat // 4
        self.parts = []
        self.sorted = None

    def append(self, pos, pat, mis):
        if self.sorted is not None:
            raise MpbError(-1, "the site list is sealed: no site can be added")
        self.parts.append((np.asarray(pos, np.uint64) << np.uint64(self.pat_bits + 4))
                          | (np.asarray(pat, np.uint64) << np.uint64(4)) | np.asarray(mis, np.uint64))

    def seal(self) -> int:
        if self.sorted is not None:
            raise MpbError(-1, "the site list is sealed already")
        self.sorted = np.sort(np.concatenate(self.parts + [np.zeros(0, np.uint64)]))
        return len(self.sorted)

    def keys(self) -> np.ndarray:
        return self.sorted.copy() if self.sorted is not None else np.concatenate(self.parts + [np.zeros(0, np.uint64)])

    def sites(self):
        """(position, pattern, mismatches, record) int64 arrays of the sealed list"""
        if self.sorted is None:
            raise MpbError(-1, "the site list is not sealed")
        k = self.sorted
        pos = (k >> np.uint64(self.pat_bits + 4)).astype(np.int64)
        pat = ((k >> np.uint64(4)) & np.uint64((1 << self.pat_bits) - 1)).astype(np.int64)
        rec = np.searchsorted(self.rec_off, pos, side="right") - 1
        return pos, pat, (k & np.uint64(15)).astype(np.int64), rec

    def _check(self, lo, hi):
        if not 0 < lo <= hi:
            raise MpbError(-1, "product lengths %d..%d: need 0 < lo <= hi" % (lo, hi))

    def cross(self, lo: int, hi: int, pair: int, eligible) -> np.ndarray:
        pos, pat, _, rec = self.sites()
        self._check(lo, hi)
        if not 0 <= pair < self.n_pairs:
            raise MpbError(-1, "pair %d outside 0..%d" % (pair, self.n_pairs - 1))
        eligible = np.asarray(eligible, bool)
        out = np.zeros(self.n_pairs, np.uint8)
        ln = self.lens[pat]
        ok = eligible[pat // 4]
        for k in np.nonzero(pat // 4 == pair)[0].tolist():
            g, p, r = int(pos[k]), int(pat[k]), int(rec[k])
            end = int(self.rec_off[r] + self.rec_len[r])
            lt, pt = int(self.lens[p]), int(PRIMER_OF[p % 4])
            if p % 2 == 0:        # right sites y of the eligible pairs
                y, q, lj = pos, pat, ln
                hit = ok & (q % 2 == 1) & (y >= g + lt) & (y + lj - g >= lo) & (y + lj - g <= hi) & (y + lj <= end)
                side = 0
            else:                 # left sites x of the eligible pairs
                x, q, li = pos, pat, ln
                hit = ok & (q % 2 == 0) & (x >= self.rec_off[r]) & (x + li <= g) & (g + lt - x >= lo) & (g + lt - x <= hi)
                side = 4
            for qq in np.unique(pat[hit]).tolist():
                out[qq // 4] |= np.uint8(1 << (side | int(PRIMER_OF[qq % 4]) << 1 | pt))
        return out

    def own(self, lo: int, hi: int) -> np.ndarray:
        pos, pat, _, rec = self.sites()
        self._check(lo, hi)
        out = np.zeros(self.n_pairs, np.uint8)
        for k in np.nonzero(pat % 2 == 0)[0].tolist():
            g, p, r = int(pos[k]), int(pat[k]), int(rec[k])
            end = int(self.rec_off[r] + self.rec_len[r])
            ll = int(self.lens[p])
            for rp in (p - p % 4 + 1, p - p % 4 + 3):
                rl = int(self.lens[rp])
                y = pos[pat == rp]
                if ((y >= g + ll) & (y + rl - g >= lo) & (y + rl - g <= hi) & (y + rl <= end)).any():
                    out[p // 4] |= np.uint8(1 << (int(PRIMER_OF[p % 4]) << 1 | int(PRIMER_OF[rp % 4])))
        return out

    def close(self):
        pass


class Msa(_Msa):
    def pattern_cover_keep(self, allow, lens, strict, v, stride, rec_off, rec_len, lo, hi, mat, row0, max_sites,
                           sites: SiteList):
        lens = np.asarray(lens, np.int64)
        rec_off = np.asarray(rec_off, np.int64)
        rec_len = np.asarray(rec_len, np.int64)
        p0 = 4 * int(row0)
        if p0 + len(lens) > len(sites.lens) or (sites.lens[p0:p0 + len(lens)] != lens).any():
            raise MpbError(-1, "patterns outside the site list or of other lengths")
        if len(rec_off) != len(sites.rec_off) or (rec_off != sites.rec_off).any() or (rec_len != sites.rec_len).any():
            raise MpbError(-1, "records differ from the site list's")
        if mat is not None:
            stats = self.pattern_cover(allow, lens, strict, v, stride, rec_off, rec_len, lo, hi, mat, row0, max_sites)
        else:
            stats = np.zeros(3, np.int64)
        if not len(rec_off):
            return stats
        hp, hr, hx, hm = (np.asarray(a, np.int64) for a in self.pattern_sites(allow, lens, strict, v))
        g = hr * stride + hx
        rec = np.searchsorted(rec_off, g, side="right") - 1
        keep = (hx < stride) & (rec >= 0)
        keep &= g + lens[hp] <= rec_off[np.maximum(rec, 0)] + rec_len[np.maximum(rec, 0)]
        if mat is None:
            stats[:] = len(hp), (keep & (hp % 2 == 0)).sum(), (keep & (hp % 2 == 1)).sum()
        sites.append(g[keep], hp[keep] + p0, hm[keep])
        return stats
