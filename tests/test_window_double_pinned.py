"""The CPU double of the window tables and the candidate scan (tests/fake_device.py: Hist, Msa.scan) pinned to the
oracle on the edge alignments of tests/edge_alignments.py, before tests/test_gpu_window_tables.py compares libmpb200
with it: table contents against oracle.tally_window, the majority seed, the base / dinucleotide tensors, and the scan
counts and row bits against a count taken per expansion with oracle.mismatch_positions and strict_positions."""
import numpy as np
import pytest

from multiprime_b200 import core
from multiprime_b200.iupac import BASES
from oracle import mp_oracle as o
from tests import edge_alignments as ea
from tests import fake_device as fd

CASES = ea.table_cases()


def _msa(case):
    return fd.Msa(None, core.pack4(case.codes), case.n, case.L, lens=case.lens)


@pytest.mark.parametrize("case", CASES, ids=str)
def test_double_tables_equal_oracle_tally(case):
    k, v = case.k, case.v
    msa = _msa(case)
    h = msa.hist(k, v, case.win_pos)
    gap_n, n_ig, n_ent = h.counts()
    st = h.stats()
    freq, nn = h.tensors(np.ones(h.nw, np.uint8))
    exc = sorted(zip(*[a.tolist() for a in h.exceptions()]))
    prm = o.Params(k=k, variation=v, fraction=-1.0)          # 1 - fraction = 2: the early gap-fraction break never fires
    ids = list(range(case.n))
    want_exc = []
    for wi, p in enumerate(case.win_pos):
        t = o.tally_window(ids, msa.rows, p, prm)
        assert not t.gap_fail
        iupac_gap = {w: c for w, c in t.gap_seq.items() if set(w) - set("ACGT-")}
        want = dict(t.cover)
        want.update({w: c for w, c in t.gap_seq.items() if w not in iupac_gap})
        got = {fd.key_string(key, k): c for key, (c, _) in h.tables[wi].items()}
        assert got == want, (case, p)
        assert gap_n[wi] == t.gap_n and case.n - gap_n[wi] == t.cover_number
        assert n_ig[wi] == sum(iupac_gap.values()) and n_ent[wi] == len(want)
        if iupac_gap:
            want_exc += [(wi, s) for s, row in enumerate(msa.rows) if o.window_kmer(row, p, k) in iupac_gap]
        gap_keys = len(want) - len(t.cover)
        assert st["nuniq"][wi].tolist() == [len(t.cover), gap_keys, len(t.cover_mm)]
        assert st["ent"][wi, 0] == sum(t.cover.values())
        assert st["ent"][wi, 2] == t.gap_n - sum(iupac_gap.values())
        if t.cover_mm:
            seed = "".join(BASES[b] for b in o.majority_seed(t.cover_mm))
            assert fd.key_string(st["mm_key"][wi], k) == seed and st["mm_cnt"][wi] == t.cover_mm[seed], (case, p)
        else:
            assert st["mm_key"][wi] == fd.KEY_EMPTY and st["mm_cnt"][wi] == 0
        f_want, _ = o.base_counts(t, k)
        assert (freq[wi] == np.array(f_want)).all(), (case, p)
        assert (nn[wi] == np.array(o.dinuc_counts(t, k))).all(), (case, p)
    assert exc == want_exc


def _mask(positions, k):
    return sum(1 << i for i in positions if 0 <= i < k)


@pytest.mark.parametrize("case", [c for c in CASES if c.n <= 4097], ids=str)
def test_double_scan_equals_mismatch_count(case):
    k, v = case.k, case.v
    msa = _msa(case)
    nw = len(case.win_pos)
    windows = sorted(set(np.linspace(0, nw - 1, min(nw, 8)).astype(int).tolist()))
    wins, allows, _ = ea.candidates(case, 17, windows)
    pos = [case.win_pos[w] for w in wins]
    words = (case.n + 31) // 32
    for fs, rs in [(set(), set()), (set(range(k)), set(range(k))), o.strict_positions("1,2,-1", k)]:
        fmask, rmask = _mask(fs, k), _mask(rs, k)
        got, bits = msa.scan(k, v, fmask, rmask, pos, allows, bits_slot=np.arange(len(pos)))
        want = np.zeros((len(pos), 3), np.int64)
        wbits = np.zeros((len(pos), 3, words), np.uint32)
        for ci, (p, allow) in enumerate(zip(pos, allows)):
            sets = [{BASES[b] for b in range(4) if (int(allow[b]) >> i) & 1} for i in range(k)]
            empty = {i for i, s in enumerate(sets) if not s}
            primer = "".join(o.SET2CODE[frozenset(s)] if s else "N" for s in sets)
            for si, row in enumerate(msa.rows):
                w = o.window_kmer(row, p, k)
                non_f = non_r = False
                isgap = w.count("-") > v
                if not isgap:
                    for hap in o.expand(w):
                        mis = set(o.mismatch_positions(primer, hap)) | empty
                        ok_f = len(mis) <= v and not mis & fs
                        ok_r = len(mis) <= v and not mis & rs
                        want[ci] += [not mis, ok_f and bool(mis), ok_r and bool(mis)]
                        non_f |= not ok_f
                        non_r |= not ok_r
                for j, flag in enumerate((non_f, non_r, isgap)):
                    if flag:
                        wbits[ci, j, si >> 5] |= np.uint32(1 << (si & 31))
        assert (got == want).all(), (case, fmask, rmask)
        assert (bits == wbits).all(), (case, fmask, rmask)
        assert want[:, 0].sum() > 0


def test_double_refuses_a_row_shorter_than_k():
    """a row with fewer than k bases cannot give a k-mer (libmpb200 returns MPB_EEXPAND; the double asserts)"""
    case = [c for c in ea.refused_cases() if c.refuse == "short"][0]
    with pytest.raises(AssertionError):
        _msa(case).hist(case.k, case.v, case.win_pos)
