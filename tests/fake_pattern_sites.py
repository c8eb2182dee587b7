"""The CPU double of mpb_pattern_sites, on top of tests/fake_device.py (its Context and Msa otherwise).

TEST INFRASTRUCTURE ONLY: pass this module as the backend of multiprime_b200.primer_coverage to run the tool's host
logic without a GPU; tests/test_gpu_pattern_sites.py pins the double to the same plain statement of the rule as the
real kernel."""
from __future__ import annotations

import numpy as np

from multiprime_b200.iupac import CODE_CHARS
from tests.fake_device import Context  # noqa: F401  (the backend's Context)
from tests.fake_device import Msa as _Msa


class Msa(_Msa):
    def pattern_sites(self, allow, lens, strict, v, max_hits=1 << 20):
        """mpb_pattern_sites: sites with at most v mismatches (a cell that is not exactly one allowed base mismatches)
        and none at a strict position, inside each row's length"""
        if not 0 <= v <= 15 or any(v >= int(ln) for ln in lens):
            raise ValueError("bad mismatch bound")
        allow = np.asarray(allow).reshape(-1, 4)
        lut = np.zeros(256, np.uint8)
        lut[np.frombuffer(CODE_CHARS.encode(), np.uint8)] = np.arange(16, dtype=np.uint8)
        rlen = np.array([len(s) for s in self.rows], np.int64)
        width = int(rlen.max()) if len(rlen) else 0
        codes = np.zeros((len(self.rows), width), np.uint8)
        for r, s in enumerate(self.rows):
            codes[r, :len(s)] = lut[np.frombuffer(s.encode(), np.uint8)]
        out = []
        for p, (al, ln) in enumerate(zip(allow, lens)):
            ln = int(ln)
            nx = width - ln + 1
            if nx <= 0:
                continue
            mis = np.zeros((len(self.rows), nx), np.int32)
            dead = np.zeros((len(self.rows), nx), bool)
            for i in range(ln):
                ok = np.zeros(16, bool)
                for b in range(4):
                    if (int(al[b]) >> i) & 1:
                        ok[1 << b] = True
                m = ~ok[codes[:, i:i + nx]]
                mis += m
                if (int(strict[p]) >> i) & 1:
                    dead |= m
            good = (mis <= v) & ~dead & (np.arange(nx)[None, :] + ln <= rlen[:, None])
            r, x = np.nonzero(good)
            out.append(np.stack([np.full(len(r), p), r, x, mis[r, x]], 1))
        a = np.concatenate(out).astype(np.int32) if out else np.zeros((0, 4), np.int32)
        return a[:, 0], a[:, 1], a[:, 2], a[:, 3]
