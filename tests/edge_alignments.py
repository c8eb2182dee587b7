"""Seeded alignments at the edges of the window passes, for the entry-point tests of the window tables and the candidate
scan (tests/test_window_double_pinned.py pins the CPU double to the oracle on them, tests/test_gpu_window_tables.py pins
libmpb200 to the double).

Every case is synth.synth_codes plus planted rows.  The shapes cross the 32-row words, the 4096-row blocks of k_hist_col
and 2^16 rows; n_col is never a multiple of 32; inputs are aligned or ragged (`lens`).  Window starts cover column 0,
p % 32 in {0, 31, 32 - k}, a dense run longer than one chunk of the column passes (33 - k starts), duplicated and
unsorted starts, p = n_col - k and starts past it (the window runs off the end of the alignment: the reference
left-extends it, core:683-687).  Cells are 4-bit base sets: A=1, C=2, G=4, T=8, IUPAC = OR of its bases, gap = 0.
"""
from __future__ import annotations

import numpy as np

A, C, G, T, R, Y, N = 1, 2, 4, 8, 5, 10, 15


class Case:
    """(codes, lens, k, v, win_pos) plus what a test should do with it: walk = batch indices worth a refinement walk,
    n_cand = random scan candidates per window, caps = log2_cap values to build the tables with besides the default"""

    def __init__(self, name, codes, lens, k, v, win_pos, walk=(), n_cand=2, caps=(), refuse=None):
        self.name, self.codes, self.lens, self.k, self.v = name, codes, lens, k, v
        self.win_pos = [int(p) for p in win_pos]
        self.walk, self.n_cand, self.caps, self.refuse = list(walk), n_cand, tuple(caps), refuse

    @property
    def n(self):
        return self.codes.shape[0]

    @property
    def L(self):
        return self.codes.shape[1]

    def __repr__(self):
        return self.name


def window_starts(L, k, rng, dense=True, n_random=4):
    """0, p % 32 in {0, 31, 32 - k}, a dense run of 33 - k + 3 starts, random starts, n_col - k and two starts past it;
    two starts repeated; the whole list shuffled"""
    pos = [p for p in (0, 31, 32 - k, 32, 63, 64 + 32 - k) if p <= L - k]
    if dense:
        a = 33 + int(rng.integers(0, 8))
        pos += [p for p in range(a, a + 33 - k + 3) if p <= L - k]
    pos += rng.integers(0, L - k + 1, n_random).tolist()
    pos += sorted({L - k, L - k + 1, L - 1})
    pos += [pos[1], pos[-1]]
    rng.shuffle(pos)
    return pos


def _random_row(rng, L):
    return (np.uint8(1) << rng.integers(0, 4, L)).astype(np.uint8)


def plant(codes, k, v, p, rows, shift=0):
    """overwrite the rows `rows` with the hard cases of the window starting at column p (kind = (i + shift) % 8 for
    the i-th row)"""
    L = codes.shape[1]
    for i, s in enumerate(rows):
        row = codes[s]
        kind = (i + shift) % 8
        if kind == 0:                                    # leading gap run longer than k, reaching into the window
            row[:k + 3] = 0
            if p < L // 2:
                row[:p + 2] = 0
        elif kind == 1:                                  # trailing gap run longer than k, from inside the window
            row[max(0, L - k - 3):] = 0
            if p + k - 2 > L // 2:
                row[p + k - 2:] = 0
        elif kind == 2:                                  # window starts and ends in gap runs, gapped flanks
            for c in (p, p + 1, p - 1, p - 3, p + k - 1, p + k - 2, p + k, p + k + 2):
                if 0 <= c < L:
                    row[c] = 0
        elif kind == 3:                                  # inner gaps only (a gap row when there are more than v)
            for c in range(p + 1, min(L, p + 1 + min(v + 1, k - 2))):
                row[c] = 0
        elif kind == 4:                                  # IUPAC cells inside the window
            for c, x in ((p + 1, N), (p + k // 2, R), (p + k - 1, Y)):
                if c < L:
                    row[c] = x
        elif kind == 5:                                  # IUPAC cell in the patching context of a leading gap
            if p >= 2:
                row[p] = 0
                row[p - 1] = Y
                row[p - 2] = 0
            if p + k + 1 < L:
                row[p + k - 1] = 0
                row[p + k + 1] = R
        elif kind == 6:                                  # gap row holding an IUPAC cell (an exception row)
            for c in range(p + 1, min(L, p + 1 + min(v + 1, k - 2))):
                row[c] = 0
            if p + k - 2 < L and v + 3 < k:
                row[p + k - 2] = N
        else:                                            # all gaps in the window, bases around it
            row[p:p + k] = 0
    return codes


def _unsupported(codes, lens, k, win_pos):
    """rows where a window needs the left extension and finds fewer than k bases left of it (the input is refused)"""
    n, L = codes.shape
    ln = np.full(n, L) if lens is None else np.asarray(lens)
    cum = np.zeros((n, L + 1), np.int32)
    np.cumsum(codes != 0, axis=1, out=cum[:, 1:])
    bad = np.zeros(n, bool)
    for p in set(win_pos):
        bad |= (p + k > ln) & (cum[np.arange(n), np.minimum(p, ln)] < k)
    return np.nonzero(bad)[0]


def _supported(codes, lens, k, win_pos, rng):
    """replace the rows _unsupported finds (synthetic rows with long gap runs at both ends) by plain random rows"""
    for s in _unsupported(codes, lens, k, win_pos):
        codes[s] = _random_row(rng, codes.shape[1])
        if lens is not None:
            codes[s, lens[s]:] = 0
    assert len(_unsupported(codes, lens, k, win_pos)) == 0


def _ragged(codes, rng, lo, k):
    """row lengths drawn from lo..n_col (every eighth row full length), but long enough that a window running past the
    row end finds the k bases of its left extension"""
    n, L = codes.shape
    lens = rng.integers(lo, L + 1, n).astype(np.int32)
    lens[rng.integers(0, n, max(1, n // 8))] = L
    kth = np.argmax(np.cumsum(codes != 0, axis=1) >= k, axis=1)          # column of each row's k-th base
    lens = np.minimum(np.maximum(lens, kth + 1 + k), L).astype(np.int32)
    for s, m in enumerate(lens):
        codes[s, m:] = 0
    return lens


def _base(n, L, seed, **kw):
    from multiprime_b200 import synth
    kw.setdefault("gap_rate", 0.01)
    kw.setdefault("iupac_rate", 0.002)
    kw.setdefault("term_gap", 0.1)
    return synth.synth_codes(n, L, seed=seed, **kw)


def _spread_rows(n, m, rng):
    """m row indices spread over words and blocks, including the first and last row and rows around 32 / 4096 / 2^16"""
    marks = [0, n - 1, 31, 32, 4095, 4096, 65535, 65536]
    out = [s for s in marks if s < n] + rng.integers(0, n, m).tolist()
    return list(dict.fromkeys(out))[:m]


def table_cases():
    """the cases every table / scan comparison runs on"""
    rng = np.random.default_rng(20261015)
    out = []

    def add(name, n, L, k, v, ragged=False, seed=1, dense=True, n_random=4, plant_at=2, walk=(), n_cand=2, **kw):
        codes = _base(n, L, seed, **kw)
        lens = None
        pos = window_starts(L, k, rng, dense=dense, n_random=n_random)
        ps = sorted(set(pos))
        for j, p in enumerate(ps[:plant_at] + ps[-plant_at:]):
            plant(codes, k, v, p, _spread_rows(n, 8, rng), shift=j)
        if ragged:
            lens = _ragged(codes, rng, max(2 * k + 12, L // 2), k)
        _supported(codes, lens, k, pos, rng)
        out.append(Case(name, codes, lens, k, v, pos, walk=walk, n_cand=n_cand))

    add("n1_k3_v0", 1, 45, 3, 0, seed=2, walk=(0, 3))
    add("n31_k5_v1_ragged", 31, 77, 5, 1, ragged=True, seed=3, walk=(1,))
    add("n33_k8_v3", 33, 71, 8, 3, seed=4, walk=(0, 5))
    add("n300_k8_v9", 300, 53, 8, 9, seed=5, gap_rate=0.08)            # variation >= k: all-gap rows are cover rows
    add("n4095_k9_v4_ragged", 4095, 67, 9, 4, ragged=True, seed=6, n_random=2)
    add("n4097_k16_v15", 4097, 99, 16, 15, seed=7, dense=False, gap_rate=0.05)
    add("n4097_k17_v1_ragged", 4097, 101, 17, 1, ragged=True, seed=8, dense=False)
    add("n500_k27_v0", 500, 95, 27, 0, seed=9, n_random=2)
    add("n70001_k18_v3", 70001, 61, 18, 3, seed=10, dense=False, n_random=0, plant_at=1, n_cand=1)

    # one clade: every row the same (one key per window, counted n times)
    row = _base(1, 70, 11, gap_rate=0.0, iupac_rate=0.0, term_gap=0.0)[0]
    codes = np.repeat(row[None, :], 300, axis=0)
    out.append(Case("identical_k18", codes, None, 18, 3, window_starts(70, 18, rng, dense=False), walk=(0,)))

    # no gap-free haplotype in window 0: every row holds one gap inside it (cover rows, v = 1)
    codes = _base(64, 40, 12, gap_rate=0.0, iupac_rate=0.0, term_gap=0.0)
    codes[np.arange(64), 11 + np.arange(64) % 3] = 0
    out.append(Case("no_gapfree_k5", codes, None, 5, 1, [10, 0, 20, 35, 38], walk=(0, 2)))

    # a hot key plus singletons: ~1500 entries per window, tables built at 2^11 slots (73 % full) and 2^10 (overflow)
    n, L, k = 3000, 40, 16
    codes = np.repeat(_base(1, L, 13, gap_rate=0.0, iupac_rate=0.0, term_gap=0.0), n, axis=0)
    r2 = np.random.default_rng(13)
    for s in range(n // 2, n):
        codes[s] = _random_row(r2, L)
    out.append(Case("hot_singletons_k16", codes, None, k, 2, [0, 5, 24, 30], n_cand=2, caps=(11, 10)))

    # one row whose window expands to exactly 65 536 haplotypes (expansion index 65 535 in `first`)
    n, L, k = 40, 64, 16
    codes = _base(n, L, 14, gap_rate=0.0, iupac_rate=0.0, term_gap=0.0)
    codes[5, 20:36:2] = N
    out.append(Case("expand_65536_k16", codes, None, k, 1, [20, 0, 48, 62], n_cand=1))
    return out


def refused_cases():
    """inputs the library refuses with MPB_EEXPAND (an error return, not a fault)"""
    out = []
    n, L, k = 40, 64, 16
    codes = _base(n, L, 15, gap_rate=0.0, iupac_rate=0.0, term_gap=0.0)
    codes[7, 20:36:2] = N
    codes[7, 21] = R                                                     # 4^8 * 2 = 131 072 expansions
    out.append(Case("expand_131072_k16", codes, None, k, 1, [0, 20], refuse="expand"))
    codes = _base(n, L, 16, gap_rate=0.0, iupac_rate=0.0, term_gap=0.0)
    lens = np.full(n, L, np.int32)
    lens[9] = k - 2                                                      # a row with fewer than k bases
    codes[9, k - 2:] = 0
    out.append(Case("short_row_k16", codes, lens, k, 1, [0, 30], refuse="short"))
    return out


def candidates(case, seed, windows=None, per_window=2):
    """scan candidates of the case (batch indices `windows`, default all): test_gpu_colscan's random ones (relaxed
    k-mers of random rows, every second one with a trial, the last one of each window with an empty position) plus one
    fully degenerate candidate -> (win, allow[nc, 4], trial)"""
    from tests.test_gpu_colscan import _random_candidates
    rng = np.random.default_rng(seed)
    windows = list(range(len(case.win_pos))) if windows is None else list(windows)
    pos = [case.win_pos[w] for w in windows]
    wins, allows, trials = _random_candidates(rng, case.codes, pos, case.k, per_window=per_window)
    wins = np.array(windows, np.int32)[wins]
    full = (1 << case.k) - 1
    wins = np.append(wins, np.int32(windows[0]))
    allows = np.vstack([allows, np.full((1, 4), full, np.uint32)])
    trials = np.append(trials, np.int32(-1))
    return wins.astype(np.int32), allows.astype(np.uint32), trials.astype(np.int32)
