"""GPU suite: libmpb200's window tables and candidate scan against the CPU double (tests/fake_device.py, pinned to the
oracle by tests/test_window_double_pinned.py), entry point by entry point, on the edge alignments of
tests/edge_alignments.py and with both window passes (MPB_WINPASS=col, the default, and row).  Exact comparisons, except
the entropy sums (`ent`, the prefilter's s1), which may differ by summation order."""
import numpy as np
import pytest

from tests import edge_alignments as ea
from tests import fake_device as fd

pytestmark = pytest.mark.gpu

CASES = ea.table_cases()
MODES = ["col", "row"]
_DOUBLE = {}                      # the double's results, once per case


def _scan_windows(case):
    nw = len(case.win_pos)
    return sorted(set(np.linspace(0, nw - 1, min(nw, 3 if case.n > 5000 else 8)).astype(int).tolist()))


def _mask_pairs(case):
    from multiprime_b200 import core
    full = (1 << case.k) - 1
    strict = core.strict_masks("1,2,-1", case.k)
    return [strict] if case.n > 5000 else [(0, 0), (full, full), strict]


def _inside(case):
    return [p for p in case.win_pos if p + case.k <= case.L]


def _fake_msa(case, rows=None, row0=0):
    from multiprime_b200 import core
    codes = case.codes if rows is None else case.codes[rows]
    lens = case.lens if rows is None or case.lens is None else case.lens[rows]
    msa = fd.Msa(None, core.pack4(codes), len(codes), case.L, lens=lens)
    msa.set_row0(row0)
    return msa


def _double(case):
    if case.name in _DOUBLE:
        return _DOUBLE[case.name]
    from multiprime_b200 import _lib
    k, v, nw = case.k, case.v, len(case.win_pos)
    msa = _fake_msa(case)
    h = msa.hist(k, v, case.win_pos)
    d = dict(counts=h.counts(), stats=h.stats(), summary=h.summary(), dumps=[h.dump(w, 0) for w in range(nw)])
    d["sel"] = (np.arange(nw) % 3 != 1).astype(np.uint8)
    d["tensors"] = h.tensors(d["sel"])
    d["tensors_all"] = h.tensors(np.ones(nw, np.uint8))
    d["exc"] = sorted(zip(*[a.tolist() for a in h.exceptions()]))
    d["seqkeys"] = msa.seqkeys(k, case.win_pos)
    d["attr"] = msa.seq_attr_hist()
    wins, allows, trials = ea.candidates(case, 23, _scan_windows(case))
    d["cands"] = _lib.make_cands(wins, allows, trials)
    d["match"] = h.match(wins, allows)
    slots = np.arange(len(wins), dtype=np.int32)
    if not case.name.startswith("expand"):
        d["scan"] = {m: h.cscan(m[0], m[1], d["cands"], bits_slot=slots) for m in _mask_pairs(case)}
    if k >= 8 and case.n <= 5000:
        ins = _inside(case)
        d["pre_row"] = msa.prefilter(k, v, case.win_pos, code="row")
        d["pre_inside"] = {code: msa.prefilter(k, v, ins, code=code) for code in ("bs", "row")}
    d["fake_h"] = h
    _DOUBLE[case.name] = d
    return d


def _gpu_msa(ctx, case, rows=None):
    from multiprime_b200 import _lib, core
    codes = case.codes if rows is None else np.ascontiguousarray(case.codes[rows])
    lens = case.lens if rows is None or case.lens is None else case.lens[rows]
    return _lib.Msa(ctx, core.pack4(codes), len(codes), case.L, lens=lens)


def _assert_stats(got, want, what):
    for name in ("gap_n", "nuniq", "mm_key", "mm_cnt", "mm_first", "n_iupac_gap"):
        assert (got[name] == want[name]).all(), (what, name)
    assert np.allclose(got["ent"], want["ent"], rtol=1e-12, atol=0), what


def _assert_dumps(h, want, n_ent, what):
    for w, (wk, wc, wf) in enumerate(want):
        gk, gc, gf = h.dump(w, int(n_ent[w]) + 1)
        assert len(gk) == len(wk), (what, w)
        assert (gk == wk).all() and (gc == wc).all() and (gf == wf).all(), (what, w)   # first-seen order included


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CASES, ids=str)
def test_tables_and_summaries(case, mode, monkeypatch):
    from multiprime_b200 import _lib
    d = _double(case)
    monkeypatch.setenv("MPB_WINPASS", mode)
    k, v, nw = case.k, case.v, len(case.win_pos)
    ctx = _lib.Context(0)
    msa = _gpu_msa(ctx, case)
    with msa.hist(k, v, case.win_pos) as h:
        counts = h.counts()
        for x, y, name in zip(counts, d["counts"], ("gap_n", "n_iupac_gap", "n_entries")):
            assert (x == y).all(), name
        _assert_dumps(h, d["dumps"], counts[2], case)
        ew, es = h.exceptions()
        assert sorted(zip(ew.tolist(), es.tolist())) == d["exc"]
        _assert_stats(h.stats(), d["stats"], "stats")
        summ = h.summary()
        _assert_stats(summ, d["summary"], "summary")
        assert (summ["freq"] == d["summary"]["freq"]).all() and (summ["nn"] == d["summary"]["nn"]).all()
        freq, nn = h.tensors(d["sel"])
        assert (freq == d["tensors"][0]).all() and (nn == d["tensors"][1]).all()
        c = d["cands"]
        assert (h.match(c["win"], c["allow"]) == d["match"]).all()
    assert (msa.seqkeys(k, case.win_pos) == d["seqkeys"]).all()
    for x, y in zip(msa.seq_attr_hist(), d["attr"]):
        assert (x == y).all()
    if "pre_row" in d:
        s0, s1 = msa.prefilter(k, v, case.win_pos)          # windows past the end: the row-domain kernel in both modes
        assert (s0 == d["pre_row"][0]).all() and np.allclose(s1, d["pre_row"][1], rtol=1e-12, atol=0)
        code = "bs" if mode == "col" and case.lens is None else "row"
        s0, s1 = msa.prefilter(k, v, _inside(case))
        w0, w1 = d["pre_inside"][code]
        assert (s0 == w0).all() and np.allclose(s1, w1, rtol=1e-12, atol=0), code
    assert d["counts"][2].sum() > 0
    msa.close()
    ctx.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", [c for c in CASES if not c.name.startswith("expand")], ids=str)
def test_scan_and_column_scan(case, mode, monkeypatch):
    """mpb_scan (row kernel) and mpb_cscan (column scan over the build's row classes): all four count columns and the
    three bit vectors, for (fmask, rmask) = (0, 0), all ones and the core's default strict positions"""
    from multiprime_b200 import _lib
    d = _double(case)
    monkeypatch.setenv("MPB_WINPASS", mode)
    k, v = case.k, case.v
    ctx = _lib.Context(0)
    msa = _gpu_msa(ctx, case)
    cands = d["cands"]
    slots = np.arange(len(cands), dtype=np.int32)
    pos = np.array(case.win_pos, np.int32)[cands["win"]]
    with msa.hist(k, v, case.win_pos) as h:
        for (fmask, rmask), (want, wbits) in d["scan"].items():
            got, gbits = h.cscan(fmask, rmask, cands, bits_slot=slots)
            assert (got == want).all(), (fmask, rmask)
            assert (gbits == wbits).all(), (fmask, rmask)
            got3, gbits3 = msa.scan(k, v, fmask, rmask, pos, cands["allow"], bits_slot=slots)
            assert (got3 == want[:, :3]).all(), (fmask, rmask)
            assert (gbits3 == wbits).all(), (fmask, rmask)
    assert sum(w[0][:, 0].sum() for w in d["scan"].values()) > 0
    msa.close()
    ctx.close()


def _cuts(n, parts):
    cuts = [0] + [n * i // parts + 5 for i in range(1, parts)] + [n]
    return [c + 1 if 0 < c < n and c % 32 == 0 else c for c in cuts]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", [c for c in CASES if c.n >= 31], ids=str)
def test_sharded_tables_equal_unsharded_double(case, mode, monkeypatch):
    """rows split into 2 and 3 shards (cuts off the 32-row grid), each with its row0: export_at -> merge_segments and
    export -> merge into empty owner tables, plus add_counts, give the unsharded double's tables, stats and tensors"""
    from multiprime_b200 import _lib
    d = _double(case)
    monkeypatch.setenv("MPB_WINPASS", mode)
    k, v, nw = case.k, case.v, len(case.win_pos)
    ones = np.ones(nw, np.uint8)
    cap = max(6, int(np.ceil(np.log2(2 * int(d["counts"][2].max()) + 64))))
    ctx = _lib.Context(0)
    full = _gpu_msa(ctx, case)
    for parts in (2, 3):
        cuts = _cuts(case.n, parts)
        shards = []
        for a, b in zip(cuts[:-1], cuts[1:]):
            m = _gpu_msa(ctx, case, rows=slice(a, b))
            m.set_row0(a)
            h = m.hist(k, v, case.win_pos)
            shards.append((m, h, h.counts()))
        gap_n = sum(c[0] for _, _, c in shards)
        n_ig = sum(c[1] for _, _, c in shards)
        parts_k, parts_c, parts_f, seg = [], [], [], [0]
        for _, h, c in shards:
            keys, cnt, first = h.export_at(np.arange(nw), c[2])
            parts_k.append(keys)
            parts_c.append(cnt)
            parts_f.append(first)
            seg += (seg[-1] + np.cumsum(c[2])).tolist()
        with full.hist(k, v, case.win_pos, log2_cap=cap, empty=True) as owner, \
                full.hist(k, v, case.win_pos, log2_cap=cap, empty=True) as owner2:
            owner.merge_segments(np.array(seg, np.int64), np.concatenate(parts_k), np.concatenate(parts_c),
                                 np.concatenate(parts_f))
            for _, h, c in shards:
                owner2.merge(*h.export(ones, c[2]))
            for o in (owner, owner2):
                o.add_counts(gap_n, n_ig)
                _assert_dumps(o, d["dumps"], d["counts"][2], (parts, "owner"))
                _assert_stats(o.stats(), d["stats"], (parts, "owner stats"))
                freq, nn = o.tensors(ones)
                assert (freq == d["tensors_all"][0]).all() and (nn == d["tensors_all"][1]).all()
        for m, h, _ in shards:
            h.close()
            m.close()
    full.close()
    ctx.close()


@pytest.mark.parametrize("mode", MODES)
def test_row0_high(mode, monkeypatch):
    """a shard at row0 = 2^40: every `first` is (row0 + s) << 16 | expansion index, as the double's"""
    from multiprime_b200 import _lib
    monkeypatch.setenv("MPB_WINPASS", mode)
    row0 = 1 << 40
    ctx = _lib.Context(0)
    for case in [c for c in CASES if c.name in ("n33_k8_v3", "n4097_k17_v1_ragged", "expand_65536_k16")]:
        rows = slice(0, min(case.n, 200))
        fh = _fake_msa(case, rows, row0).hist(case.k, case.v, case.win_pos)
        m = _gpu_msa(ctx, case, rows)
        m.set_row0(row0)
        with m.hist(case.k, case.v, case.win_pos) as h:
            n_ent = h.counts()[2]
            want = [fh.dump(w, 0) for w in range(len(case.win_pos))]
            _assert_dumps(h, want, n_ent, case)
            for w in range(len(case.win_pos)):
                first = h.dump(w, int(n_ent[w]) + 1)[2]
                assert ((first >> np.uint64(16)) >= row0).all() and ((first >> np.uint64(16)) < row0 + 200).all()
            if case.name.startswith("expand_65536"):
                assert any(((h.dump(w, int(n_ent[w]) + 1)[2] & np.uint64(0xFFFF)) == 65535).any()
                           for w in range(len(case.win_pos)))
        m.close()
    ctx.close()


@pytest.mark.parametrize("mode", MODES)
def test_small_table_rebuilds(mode, monkeypatch):
    """a hot key plus ~1500 singletons: tables of 2^11 slots (73 % full) and 2^10 slots (full: Msa.hist doubles the
    capacity and builds again) equal the double"""
    from multiprime_b200 import _lib
    monkeypatch.setenv("MPB_WINPASS", mode)
    case = [c for c in CASES if c.caps][0]
    d = _double(case)
    assert d["counts"][2].max() > 1 << 10
    ctx = _lib.Context(0)
    msa = _gpu_msa(ctx, case)
    for cap in case.caps:
        with msa.hist(case.k, case.v, case.win_pos, log2_cap=cap) as h:
            assert h.log2_cap >= cap and (h.log2_cap > cap) == (cap == 10)
            _assert_dumps(h, d["dumps"], d["counts"][2], cap)
            _assert_stats(h.stats(), d["stats"], cap)
    msa.close()
    ctx.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", [c for c in CASES if c.walk], ids=str)
def test_device_walk_equals_host_walk_on_double(case, mode, monkeypatch):
    """the device walk (WalkDev over mpb_cscan) against the host mpb_walk driven by the double's scan, same inputs"""
    from multiprime_b200 import _lib, core
    d = _double(case)
    monkeypatch.setenv("MPB_WINPASS", mode)
    fmask, rmask = core.strict_masks("1,2,-1", case.k)
    win = np.array(case.walk, np.int32)
    cover = (case.n - d["counts"][0][win]).astype(np.int64)
    mm_key = d["stats"]["mm_key"][win]
    want = d["fake_h"].walk(4, 64, fmask, rmask, win, cover, mm_key)
    ctx = _lib.Context(0)
    msa = _gpu_msa(ctx, case)
    with msa.hist(case.k, case.v, case.win_pos) as h:
        h.tensors(np.ones(len(case.win_pos), np.uint8))                    # the walk reads the tensors of the handle
        got = h.walk(4, 64, fmask, rmask, win, cover, mm_key)
    for name in ("sets", "counts", "seeds", "seed_cover", "ntracks", "trace_off"):
        assert (got[name] == want[name]).all(), name
    n_tr = int(want["trace_off"][-1])
    assert (got["trace"][:n_tr] == want["trace"][:n_tr]).all()
    msa.close()
    ctx.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", ea.refused_cases(), ids=str)
def test_refused_inputs(case, mode, monkeypatch):
    """a window of one row with 131 072 expansions, a row with fewer than k bases: MPB_EEXPAND, an error return"""
    from multiprime_b200 import _lib
    monkeypatch.setenv("MPB_WINPASS", mode)
    ctx = _lib.Context(0)
    msa = _gpu_msa(ctx, case)
    with pytest.raises(_lib.MpbError) as e:
        msa.hist(case.k, case.v, case.win_pos)
    assert e.value.code == -5
    if case.refuse == "expand":
        with msa.hist(case.k, case.v, list(range(40, 48))) as h:          # the alignment stays usable
            assert h.counts()[2].min() > 0
    msa.close()
    ctx.close()
