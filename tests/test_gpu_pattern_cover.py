"""mpb_pattern_cover, mpb_cover_gains and mpb_cover_take against the CPU double (tests/fake_pattern_cover.py) and against
primer_coverage.amplicons on the same panel: a bit is set exactly where the pair has an amplicon, and the perfect bit
exactly where the best amplicon has no mismatch.  The gains against numpy popcounts at the word edges."""
import ctypes as C

import numpy as np
import pytest

from tests.test_primer_coverage import make_case

pytestmark = pytest.mark.gpu


def _panel(tmp_path, seed, n_extra=0):
    from multiprime_b200 import primer_coverage as pc
    from multiprime_b200.pcr_product import parse_primers
    fa, pf, lo, hi = make_case(tmp_path, seed)
    pairs = dict(parse_primers(pf, "fa"))
    names = list(pairs)
    for k in range(n_extra):                           # more rows: the same pairs again, swapped F / R
        f, r = pairs[names[k % len(names)]]
        pairs["extra%d" % k] = (r, f) if k % 2 else (f, r)
    return pc.read_targets(fa), pc.Panel(pairs, "1,2,-1"), lo, hi


def _build(backend, targets, panel, v, lo, hi, a, b, block):
    """the matrix of the records [a, b) built in blocks of `block` pairs -> (amp, perf) host arrays, stats"""
    from multiprime_b200 import primer_coverage as pc
    n = len(panel.names)
    rows, width, starts = pc.layout(targets, panel.lmax)
    end = int(starts[b - 1] + targets.lens[b - 1])
    row0 = int(starts[a]) // pc.S
    row1 = max(row0 + 1, -(-end // pc.S))
    ctx = backend.Context.shared(0)
    mat = backend.CoverMatrix(ctx, n, b - a)
    msa = backend.Msa(ctx, rows[row0:row1], row1 - row0, width, row_bytes=rows.shape[1])
    stats = np.zeros(3, np.int64)
    try:
        for p0 in range(0, n, block):
            p1 = min(n, p0 + block)
            stats += msa.pattern_cover(panel.allow[4 * p0:4 * p1], panel.plen[4 * p0:4 * p1],
                                       panel.strict[4 * p0:4 * p1], v, pc.S, starts[a:b] - row0 * pc.S,
                                       targets.lens[a:b], lo, hi, mat, p0)
        amp, perf, cov, covp = mat.to_host()
    finally:
        msa.close()
        mat.close()
    assert not cov.any() and not covp.any()
    return amp, perf, stats


def _bits(mat_rows, n_rec):
    return np.unpackbits(mat_rows.view(np.uint8), axis=-1, bitorder="little")[:, :n_rec].astype(bool)


def _want(targets, panel, v, lo, hi):
    """amp / perf [pairs, records] from primer_coverage's own pairing"""
    from multiprime_b200 import primer_coverage as pc
    from tests import fake_pattern_sites
    best = pc.amplicons(pc.find_sites(targets, panel, v, backend=fake_pattern_sites), panel, targets.lens, lo, hi, v)
    n_rec = len(targets.names)
    amp = np.zeros((len(panel.names), n_rec), bool)
    perf = np.zeros_like(amp)
    for q, bq in enumerate(best):
        amp[q, bq["rec"]] = True
        perf[q, bq["rec"][(bq["fmis"] + bq["rmis"]) == 0]] = True
    return amp, perf


@pytest.mark.parametrize("stride", [64, None])
@pytest.mark.parametrize("v", [0, 1, 3])
def test_matrix_equals_double_and_amplicons(tmp_path, monkeypatch, stride, v):
    from multiprime_b200 import _lib
    from multiprime_b200 import primer_coverage as pc
    from tests import fake_pattern_cover
    if stride:
        monkeypatch.setattr(pc, "S", stride)
    targets, panel, lo, hi = _panel(tmp_path, v + 20, n_extra=3)
    n_rec = len(targets.names)
    assert n_rec % 32
    want_amp, want_perf = _want(targets, panel, v, lo, hi)
    assert want_amp.any() and (want_amp & ~want_perf).any() == (v > 0)
    amp_d, perf_d, stats_d = _build(fake_pattern_cover, targets, panel, v, lo, hi, 0, n_rec, len(panel.names))
    for block in (len(panel.names), 1, 4):
        amp, perf, stats = _build(_lib, targets, panel, v, lo, hi, 0, n_rec, block)
        assert (amp == amp_d).all() and (perf == perf_d).all()
        assert (_bits(amp, n_rec) == want_amp).all()
        assert (_bits(perf, n_rec) == want_perf).all()
        assert not _bits(amp, amp.shape[1] * 32)[:, n_rec:].any()
        if block == len(panel.names):
            assert (stats == stats_d).all()


@pytest.mark.parametrize("world", [2, 3])
def test_record_shards_are_column_blocks(tmp_path, monkeypatch, world):
    """the records of a rank's shard (a row straddling two shards is searched by both) give the columns of those
    records"""
    from multiprime_b200 import _lib
    from multiprime_b200 import primer_coverage as pc
    from multiprime_b200 import primer_specificity as ps
    monkeypatch.setattr(pc, "S", 64)
    targets, panel, lo, hi = _panel(tmp_path, 31)
    n_rec = len(targets.names)
    want_amp, want_perf = _want(targets, panel, 2, lo, hi)
    bounds = ps.shard_records(targets, panel.lmax, world)
    for a, b in zip(bounds[:-1].tolist(), bounds[1:].tolist()):
        if b > a:
            amp, perf, _ = _build(_lib, targets, panel, 2, lo, hi, a, b, 2)
            assert (_bits(amp, b - a) == want_amp[:, a:b]).all()
            assert (_bits(perf, b - a) == want_perf[:, a:b]).all()
    assert n_rec == bounds[-1]


def _popcount(a):
    return np.unpackbits(a.view(np.uint8), axis=-1).sum(axis=-1).astype(np.int64)


@pytest.mark.parametrize("n_rec", [1, 31, 32, 33, 100, 129, 1000])
def test_gains_and_take_against_numpy(n_rec):
    from multiprime_b200 import _lib
    rng = np.random.default_rng(n_rec)
    ctx = _lib.Context.shared(0)
    n_rows = 37
    words = _lib.words_of(n_rec)
    used = -(-n_rec // 32)
    mask = np.zeros(words, np.uint32)
    mask[:used] = 0xFFFFFFFF
    if n_rec % 32:
        mask[used - 1] = (1 << (n_rec % 32)) - 1
    amp = rng.integers(0, 1 << 32, (n_rows, words), dtype=np.uint64).astype(np.uint32) & mask
    perf = amp & rng.integers(0, 1 << 32, (n_rows, words), dtype=np.uint64).astype(np.uint32)
    mat = _lib.CoverMatrix(ctx, n_rows, n_rec)
    try:
        host = np.zeros((2 * n_rows + 2, words), np.uint32)
        host[:n_rows], host[n_rows:2 * n_rows] = amp, perf
        _lib.check(_lib.load().mpb_ctx_memcpy(ctx.h, C.c_void_p(mat.buf.p), _lib.ptr(host), host.nbytes))
        cov, covp = np.zeros(words, np.uint32), np.zeros(words, np.uint32)
        for cand in (np.arange(n_rows), np.array([5, 5, 0, 36, 17]), np.array([], np.int64), np.array([36])):
            g = ctx.cover_gains(mat, cand)
            assert g.shape == (len(cand), 2)
            assert (g[:, 0] == _popcount(amp[cand] & ~cov)).all()
            assert (g[:, 1] == _popcount(perf[cand] & ~covp)).all()
        for row in (3, 36, 0):
            ctx.cover_take(mat, row)
            cov |= amp[row]
            covp |= perf[row]
            got = mat.to_host()
            assert (got[2] == cov).all() and (got[3] == covp).all()
            g = ctx.cover_gains(mat, np.arange(n_rows))
            assert (g[:, 0] == _popcount(amp & ~cov)).all()
            assert (g[:, 1] == _popcount(perf & ~covp)).all()
        with pytest.raises(_lib.MpbError, match="outside"):
            ctx.cover_gains(mat, [n_rows])
        with pytest.raises(_lib.MpbError, match="outside"):
            ctx.cover_gains(mat, [-1])
        with pytest.raises(_lib.MpbError, match="outside"):
            ctx.cover_take(mat, n_rows)
    finally:
        mat.close()


def test_refusals(tmp_path):
    """limits come back as MPB_EINVAL with a message"""
    from multiprime_b200 import _lib
    from multiprime_b200 import primer_coverage as pc
    lib = _lib.load()
    ctx = _lib.Context.shared(0)
    mat = _lib.CoverMatrix(ctx, 4, 40)
    host = np.zeros((10, mat.words), np.uint32)
    gains = np.zeros(2, np.int64)
    cand = np.zeros(1, np.int32)
    try:
        rc = lib.mpb_cover_gains(ctx.h, C.c_void_p(mat.amp), C.c_void_p(mat.perf), 4, 6, C.c_void_p(mat.covered),
                                 C.c_void_p(mat.covered_perfect), _lib.ptr(cand), 1, _lib.ptr(gains))
        assert rc == -1 and b"multiple of 4" in lib.mpb_last_error()
        rc = lib.mpb_cover_gains(ctx.h, _lib.ptr(host), C.c_void_p(mat.perf), 4, mat.words, C.c_void_p(mat.covered),
                                 C.c_void_p(mat.covered_perfect), _lib.ptr(cand), 1, _lib.ptr(gains))
        assert rc == -1 and b"device memory" in lib.mpb_last_error()
        rc = lib.mpb_cover_take(ctx.h, C.c_void_p(mat.amp + 4), C.c_void_p(mat.perf), 4, mat.words, 0,
                                C.c_void_p(mat.covered), C.c_void_p(mat.covered_perfect))
        assert rc == -1 and b"aligned" in lib.mpb_last_error()
        targets, panel, lo, hi = _panel(tmp_path, 3)
        rows, width, starts = pc.layout(targets, panel.lmax)
        msa = _lib.Msa(ctx, rows, len(rows), width, row_bytes=rows.shape[1])
        short = _lib.Msa(ctx, rows[:2], 2, width, row_bytes=rows.shape[1])     # the last records end past its rows
        stats = np.zeros(3, np.int64)
        try:
            def call(n_pat=8, lo_=lo, hi_=hi, words=mat.words, amp=mat.amp, n_rec=len(starts), stride=pc.S,
                     max_sites=0, h=msa.h):
                return lib.mpb_pattern_cover(h, n_pat, _lib.ptr(np.ascontiguousarray(panel.allow[:8])),
                                             _lib.ptr(panel.plen[:8].copy()), _lib.ptr(panel.strict[:8].copy()), 1,
                                             stride, n_rec, _lib.ptr(starts.astype(np.int64)),
                                             _lib.ptr(targets.lens.astype(np.int64)), lo_, hi_, words,
                                             C.c_void_p(amp), C.c_void_p(mat.perf), max_sites, _lib.ptr(stats))
            for kw, msg in ((dict(n_pat=6), b"four per pair"), (dict(lo_=hi + 1), b"0 < lo <= hi"),
                            (dict(lo_=0), b"0 < lo <= hi"), (dict(words=0), b"fewer than"),
                            (dict(amp=host.ctypes.data), b"device memory"), (dict(stride=1 << 59), b"64 bits"),
                            (dict(n_rec=-1), b"n_rec"), (dict(max_sites=-1), b"max_sites"),
                            (dict(max_sites=(1 << 31) + 1), b"max_sites"), (dict(h=short.h), b"past the")):
                assert call(**kw) == -1, kw
                assert msg in lib.mpb_last_error(), (kw, lib.mpb_last_error())
            assert call() == 0
        finally:
            msa.close()
            short.close()
        with pytest.raises(_lib.MpbError):            # the matrix is 4 pairs x 40 records
            msa2 = _lib.Msa(ctx, rows, len(rows), width, row_bytes=rows.shape[1])
            try:
                msa2.pattern_cover(panel.allow[:8], panel.plen[:8], panel.strict[:8], 1, pc.S, starts, targets.lens, lo,
                                   hi, mat, 3)
            finally:
                msa2.close()
    finally:
        mat.close()


@pytest.mark.parametrize("max_sites", [1, 0, 1 << 20])
def test_search_runs_once_when_the_capacity_holds_the_sites(tmp_path, max_sites):
    """a capacity smaller than the sites takes the second search (regrow) and gives the same bits; one that holds them
    searches once"""
    from multiprime_b200 import _lib
    from multiprime_b200 import primer_coverage as pc
    targets, panel, lo, hi = _panel(tmp_path, 5, n_extra=2)
    n, n_rec = len(panel.names), len(targets.names)
    want_amp, want_perf = _want(targets, panel, 1, lo, hi)
    rows, width, starts = pc.layout(targets, panel.lmax)
    ctx = _lib.Context.shared(0)
    mat = _lib.CoverMatrix(ctx, n, n_rec)
    msa = _lib.Msa(ctx, rows, len(rows), width, row_bytes=rows.shape[1])
    try:
        ctx.profile_read(None)
        ctx.profile(True)
        stats = msa.pattern_cover(panel.allow, panel.plen, panel.strict, 1, pc.S, starts, targets.lens, lo, hi, mat, 0,
                                  max_sites)
        launches = ctx.profile_read("k_pattern_sites")[1]
        ctx.profile(False)
        amp, perf, _, _ = mat.to_host()
    finally:
        ctx.profile(False)
        msa.close()
        mat.close()
    assert stats[0] > 1
    assert launches == (2 if 0 < max_sites < stats[0] else 1)
    assert (_bits(amp, n_rec) == want_amp).all() and (_bits(perf, n_rec) == want_perf).all()
