"""mpb_site_list, mpb_pattern_cover_keep, mpb_sites_cross and mpb_sites_own against the CPU double
(tests/fake_site_list.py): the sealed list entry by entry across appended blocks, the cross and own bits on the sites of
a panel, on random sites and on dense windows where every site has hundreds of partners, the window edges (exactly lo
and hi, y = x + L_i, a window clipped at a record end), and the refusals."""
import numpy as np
import pytest

from tests.test_gpu_pattern_cover import _panel

pytestmark = pytest.mark.gpu


def _lists(targets, panel, v, lo, hi, block):
    """the GPU list (kept in blocks of `block` pairs, with the matrix) and the double's (one block) of all records"""
    from multiprime_b200 import _lib
    from multiprime_b200 import primer_coverage as pc
    from tests import fake_site_list
    n = len(panel.names)
    rows, width, starts = pc.layout(targets, panel.lmax)
    n_rec = len(targets.names)
    row1 = max(1, -(-int(starts[-1] + targets.lens[-1]) // pc.S))
    out = []
    for backend, blk in ((_lib, block), (fake_site_list, n)):
        ctx = backend.Context.shared(0)
        mat = backend.CoverMatrix(ctx, n, n_rec)
        msa = backend.Msa(ctx, rows[:row1], row1, width, row_bytes=rows.shape[1])
        sites = backend.SiteList(ctx, panel.plen, row1 * pc.S, starts, targets.lens)
        try:
            for p0 in range(0, n, blk):
                p1 = min(n, p0 + blk)
                msa.pattern_cover_keep(panel.allow[4 * p0:4 * p1], panel.plen[4 * p0:4 * p1],
                                       panel.strict[4 * p0:4 * p1], v, pc.S, starts, targets.lens, lo, hi,
                                       mat if p0 % 2 == 0 else None, p0, 0, sites)
            sites.seal()
            amp = mat.to_host()[0]
        finally:
            msa.close()
            mat.close()
        out.append((sites, amp))
    return out


@pytest.mark.parametrize("block", [1, 2, 5])
def test_sealed_list_and_joins_equal_double(tmp_path, monkeypatch, block):
    from multiprime_b200 import primer_coverage as pc
    monkeypatch.setattr(pc, "S", 64)
    targets, panel, lo, hi = _panel(tmp_path, 41, n_extra=3)
    (gpu, amp), (dbl, amp_d) = _lists(targets, panel, 2, lo, hi, block)
    try:
        keys = gpu.keys()
        assert len(keys) > 100 and (keys == dbl.keys()).all()
        assert (np.diff(keys.astype(np.uint64)) > 0).all()
        n = len(panel.names)
        rows_with_matrix = [q for q in range(n) if (q // block) % 2 == 0]
        assert (amp[rows_with_matrix] == amp_d[rows_with_matrix]).all()
        rng = np.random.default_rng(block)
        for lo2, hi2 in ((lo, hi), (40, 200), (1, 5000)):
            assert (gpu.own(lo2, hi2) == dbl.own(lo2, hi2)).all()
            for t in range(n):
                el = rng.random(n) < 0.7
                el[t] = False
                got, want = gpu.cross(lo2, hi2, t, el), dbl.cross(lo2, hi2, t, el)
                assert (got == want).all(), (lo2, hi2, t)
        assert gpu.own(lo, hi).any() and any(gpu.cross(1, 5000, t, np.ones(n, bool)).any() for t in range(n))
    finally:
        gpu.close()


def _placed(rng, n_pairs, n_rec, rec_len, per_rec, dense_window):
    """(targets FASTA text, pairs): records of random bases with the F / R of each pair planted as exact sites
    (left sites as the primer itself, right sites as its reverse complement); dense_window packs many sites of
    many pairs into the first few hundred bases of record 0"""
    from tests.test_primer_coverage import rc
    alphabet = np.array(list("ACGT"))
    primers = ["".join(rng.choice(alphabet, int(rng.integers(16, 23)))) for _ in range(2 * n_pairs)]
    recs = []
    for r in range(n_rec):
        s = list("".join(rng.choice(alphabet, rec_len)))
        k = per_rec * (6 if dense_window and r == 0 else 1)
        span = 400 if dense_window and r == 0 else rec_len
        for _ in range(k):
            i = int(rng.integers(0, 2 * n_pairs))
            site = primers[i] if rng.random() < 0.5 else rc(primers[i])
            x = int(rng.integers(0, max(1, min(span, rec_len) - len(site))))
            s[x:x + len(site)] = list(site)
        recs.append("".join(s))
    pairs = {"p%d" % q: (primers[2 * q], primers[2 * q + 1]) for q in range(n_pairs)}
    return "".join(">r%d\n%s\n" % (k, s) for k, s in enumerate(recs)), pairs


@pytest.mark.parametrize("dense", [False, True])
def test_joins_on_planted_sites_equal_double(tmp_path, monkeypatch, dense):
    """many planted sites per record (dense: hundreds of partners per window), v = 0 and 2, exact lo / hi edges taken
    from the planted products"""
    from multiprime_b200 import primer_coverage as pc
    monkeypatch.setattr(pc, "S", 512)
    rng = np.random.default_rng(7 + dense)
    text, pairs = _placed(rng, 24, 9, 3000, 60, dense)
    fa = tmp_path / "planted.fa"
    fa.write_text(text)
    targets = pc.read_targets(str(fa))
    panel = pc.Panel(pairs, "1,2,-1")
    n = len(panel.names)
    for v in (0, 2):
        (gpu, _), (dbl, _) = _lists(targets, panel, v, 20, 2000, 7)
        try:
            assert (gpu.keys() == dbl.keys()).all()
            pos, pat, _, _ = dbl.sites()
            # window edges: lo / hi equal to actual products (a left site and a right site of the same record)
            left, right = pos[pat % 2 == 0], pos[pat % 2 == 1]
            d = (right[None, :] - left[:, None])
            d = d[(d > 30) & (d < 2000)]
            edges = [(int(d.min()) + 20, int(d.max()) + 16), (int(np.median(d)), int(np.median(d)) + 22), (1, 40)]
            for lo, hi in edges:
                assert (gpu.own(lo, hi) == dbl.own(lo, hi)).all()
                for t in range(0, n, 3):
                    el = rng.random(n) < 0.8
                    el[t] = False
                    assert (gpu.cross(lo, hi, t, el) == dbl.cross(lo, hi, t, el)).all(), (v, lo, hi, t)
            if dense:
                assert sum(bin(int(b)).count("1") for b in gpu.cross(1, 2000, 0, np.arange(n) != 0)) >= 8
        finally:
            gpu.close()


def test_window_edges_exactly(tmp_path, monkeypatch):
    """X's F at x = 10 of record a with a right site at y = x + L (product 40) and one at exactly hi = 300; X's F at 0 of
    record b with a right site that ends where b ends; record c ends one base into the last right site (cut)"""
    from multiprime_b200 import primer_coverage as pc
    from tests.test_primer_coverage import rc
    monkeypatch.setattr(pc, "S", 256)
    rng = np.random.default_rng(3)

    def rand(k):
        return "".join(rng.choice(list("ACGT"), k))
    fx, ra, rb, rd, re = (rand(20) for _ in range(5))
    rec_a = rand(10) + fx + rc(ra) + rand(240) + rc(rb) + rand(5)
    rec_b = fx + rand(100) + rc(rd)
    rec_c = fx + rand(100) + rc(re)[:19]
    fa = tmp_path / "edges.fa"
    fa.write_text(">a\n%s\n>b\n%s\n>c\n%s\n" % (rec_a, rec_b, rec_c))
    pairs = {"X": (fx, rand(20)), "a": (rand(20), ra), "b": (rand(20), rb), "d": (rand(20), rd), "e": (rand(20), re)}
    targets = pc.read_targets(str(fa))
    panel = pc.Panel(pairs, "1,2,-1")
    (gpu, _), (dbl, _) = _lists(targets, panel, 0, 40, 300, 2)
    try:
        el = np.array([False, True, True, True, True])
        for lo, hi in ((40, 300), (41, 300), (40, 299)):
            assert (gpu.cross(lo, hi, 0, el) == dbl.cross(lo, hi, 0, el)).all()
        # side 0 (X's primer on the left), candidate primer R (1), X's primer F (0): bit 0b010, byte 4
        assert gpu.cross(40, 300, 0, el).tolist() == [0, 4, 4, 4, 0]
        assert gpu.cross(41, 300, 0, el).tolist() == [0, 0, 4, 4, 0]
        assert gpu.cross(40, 299, 0, el).tolist() == [0, 4, 0, 4, 0]
        # the same products seen from the candidates' right sites: X's F is the left site of each (side 1 when a
        # candidate is taken and X is eligible)
        assert gpu.cross(40, 300, 1, ~np.eye(5, dtype=bool)[1]).tolist() == [1 << (4 | 0 << 1 | 1), 0, 0, 0, 0]
    finally:
        gpu.close()


def test_refusals():
    from multiprime_b200 import _lib
    ctx = _lib.Context.shared(0)
    lens = np.full(8, 20, np.int32)
    with pytest.raises(_lib.MpbError, match="64 bits"):
        _lib.SiteList(ctx, np.full(1 << 16, 20, np.int32), 1 << 45, [0], [10])
    with pytest.raises(_lib.MpbError, match="four per pair"):
        _lib.SiteList(ctx, lens[:6], 1000, [0], [10])
    with pytest.raises(_lib.MpbError, match="past the"):
        _lib.SiteList(ctx, lens, 1000, [0, 900], [10, 200])
    s = _lib.SiteList(ctx, lens, 1000, [0], [500])
    try:
        with pytest.raises(_lib.MpbError, match="not sealed"):
            s.cross(10, 100, 0, np.ones(2, bool))
        with pytest.raises(_lib.MpbError, match="not sealed"):
            s.own(10, 100)
        assert s.seal() == 0
        with pytest.raises(_lib.MpbError, match="sealed already"):
            s.seal()
        with pytest.raises(_lib.MpbError, match="pair 2 outside 0..1"):
            s.cross(10, 100, 2, np.ones(2, bool))
        with pytest.raises(_lib.MpbError, match="0 < lo <= hi"):
            s.own(100, 10)
        assert s.cross(10, 100, 1, np.ones(2, bool)).tolist() == [0, 0] and s.own(10, 100).tolist() == [0, 0]
    finally:
        s.close()
    lib = _lib.load()
    stats = np.zeros(3, np.int64)
    rc = lib.mpb_pattern_cover_keep(None, 4, None, None, None, 0, 64, 0, None, None, 10, 100, 0, None, None, 0,
                                    _lib.ptr(stats), None, 0)
    assert rc == -1 and "NULL" in lib.mpb_last_error().decode()
