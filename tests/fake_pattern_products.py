"""The CPU double of mpb_pattern_products, on top of tests/fake_pattern_sites.py (its search and its Context / Msa).

TEST INFRASTRUCTURE ONLY: pass this module as the backend of multiprime_b200.primer_specificity to run the tool's host
logic (sharding, capping, writing) without a GPU; tests/test_gpu_pattern_products.py pins the double to the real entry
point.  The chunk budget only bounds device memory, so the double ignores it."""
from __future__ import annotations

import numpy as np

from multiprime_b200._lib import MpbError
from tests.fake_pattern_sites import Context  # noqa: F401  (the backend's Context)
from tests.fake_pattern_sites import Msa as _Msa


class Msa(_Msa):
    def pattern_products(self, allow, lens, strict, v, pat_primer, pat_side, n_primer, stride, rec_off, rec_len, lo, hi,
                         listed, max_rows, chunk=0):
        if not 1 <= n_primer <= 1024:
            raise MpbError(-1, "%d primers: at most 1024 primers are supported" % n_primer)
        if not 0 < lo <= hi <= (1 << 23) - 1:
            raise MpbError(-1, "product lengths %d..%d: need 0 < lo <= hi <= %d" % (lo, hi, (1 << 23) - 1))
        rec_off = np.asarray(rec_off, np.int64)
        rec_len = np.asarray(rec_len, np.int64)
        if len(rec_len) and (rec_len.max() > 0xFFFFFFFF or rec_len.min() < 0):
            raise MpbError(-1, "record length outside 0..4294967295 (the packed product start)")
        lens = np.asarray(lens, np.int64)
        pat_primer = np.asarray(pat_primer, np.int64)
        pat_side = np.asarray(pat_side, np.int64)
        listed = np.asarray(listed).reshape(n_primer, n_primer) != 0
        comb = np.zeros((n_primer, n_primer, 3), np.int64)
        stats = np.zeros(4, np.int64)
        empty = dict(comb=comb, union=np.zeros(2, np.int64), rows=np.zeros((0, 8), np.int64), n_listed=0, stats=stats)
        if not len(rec_off):
            return empty
        hp, hr, hx, hm = (np.asarray(a, np.int64) for a in self.pattern_sites(allow, lens, strict, v))
        stats[0] = len(hp)
        g = hr * stride + hx
        rec = np.searchsorted(rec_off, g, side="right") - 1
        keep = (hx < stride) & (rec >= 0)
        rec = np.maximum(rec, 0)
        keep &= g + lens[hp] <= rec_off[rec] + rec_len[rec]
        hp, rec, pos, mis = hp[keep], rec[keep], (g - rec_off[rec])[keep], hm[keep]
        prim, left = pat_primer[hp], pat_side[hp] == 0
        plen = np.zeros(n_primer, np.int64)
        plen[pat_primer] = lens
        stats[1], stats[2] = left.sum(), (~left).sum()
        big = int(rec_len.max()) + hi + 1
        lrec, li, lx, lm = rec[left], prim[left], pos[left], mis[left]
        o = np.argsort(rec[~left] * big + pos[~left], kind="stable")
        rrec, rj, ry, rm = rec[~left][o], prim[~left][o], pos[~left][o], mis[~left][o]
        rkey = rrec * big + ry
        q0 = np.searchsorted(rkey, lrec * big + lx + plen[li], side="left")
        q1 = np.searchsorted(rkey, lrec * big + lx + hi, side="right")
        cnt = np.maximum(q1 - q0, 0)
        a = np.repeat(np.arange(len(lx)), cnt)
        b = q0[a] + np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        length = ry[b] + plen[rj[b]] - lx[a]
        ok = (rrec[b] == lrec[a]) & (ry[b] >= lx[a] + plen[li[a]]) & (length >= lo) & (length <= hi)
        a, b, length = a[ok], b[ok], length[ok]
        if not len(a):
            return empty
        key = (lrec[a] * n_primer + li[a]) * n_primer + rj[b]
        tot = lm[a] + rm[b]
        order = np.lexsort((lx[a], length, tot, key))
        ukey, first, count = np.unique(key[order], return_index=True, return_counts=True)
        pick = order[first]
        grec, gi, gj = ukey // (n_primer * n_primer), (ukey // n_primer) % n_primer, ukey % n_primer
        perfect = tot[pick] == 0
        np.add.at(comb, (gi, gj, 0), count)
        np.add.at(comb, (gi, gj, 1), 1)
        np.add.at(comb, (gi, gj, 2), perfect.astype(np.int64))
        stats[3] = len(ukey)
        lst = listed[gi, gj]
        union = np.array([len(np.unique(grec[lst])), len(np.unique(grec[lst & perfect]))], np.int64)
        rows = np.stack([grec, gi, gj, lx[a][pick], length[pick], lm[a][pick], rm[b][pick], count], 1)[lst]
        return dict(comb=comb, union=union, rows=rows[:max_rows], n_listed=int(lst.sum()), stats=stats)
