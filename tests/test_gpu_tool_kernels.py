"""The kernels behind the other drop-in tools against plain references of the same operation:

* mpb_pattern_hits (extract_PCR_product): a numpy search of every line, at row counts that are not a multiple of 32
  or 128, ragged rows, a line wider than 65535 columns, IUPAC / N / gap cells in rows and inside planted sites, and
  more hits than the default output capacity;
* mpb_pair_cover / mpb_pair_cover3 (get_multiPrime): numpy popcounts, from host arrays and from HBM, and the padding
  bits of the scan's bit vectors;
* mpb_dimer_grid (finDimer): the 5-mer prefilter loses no pair that k_dimer_pairs finds on the full pair list."""
import ctypes as C

import numpy as np
import pytest

SINGLE = np.array([1, 2, 4, 8], np.uint8)                       # 4-bit sets of A, C, G, T
MULTI = np.array([0, 3, 5, 6, 7, 9, 10, 11, 12, 13, 14, 15], np.uint8)   # gap and every IUPAC code (N = 15)


# ---------------------------------------------------------------------------------------------------------------
# pattern search
# ---------------------------------------------------------------------------------------------------------------
def reference_hits(codes, lens, allow, plens, exact=True):
    """every (pattern, row, position) where each of the pattern's cells holds exactly one base and that base is
    allowed at that position; cells at or past lens[row] do not exist -> int64[n, 3] sorted.  exact=False lets a
    cell match when ANY of its bases is allowed (what an OR of the allowed bases' planes computes)"""
    n, width = codes.shape
    c = np.where(np.arange(width)[None, :] < np.asarray(lens)[:, None], codes, 0)
    single = np.zeros(16, bool)
    single[SINGLE] = True
    out = []
    for p, L in enumerate(plens):
        L = int(L)
        if L > width:
            continue
        ok = np.ones((n, width - L + 1), bool)
        for i in range(L):
            allowed = sum(((int(allow[p][q]) >> i) & 1) << q for q in range(4))
            tab = (np.arange(16) & allowed) != 0
            if exact:
                tab &= single
            ok &= tab[c[:, i:width - L + 1 + i]]
        r, x = np.nonzero(ok)
        out.append(np.stack([np.full(len(r), p), r, x], 1))
    return np.concatenate(out).astype(np.int64) if out else np.zeros((0, 3), np.int64)


def _expansion(rng, sets):
    return np.array([SINGLE[rng.choice([q for q in range(4) if (s >> q) & 1])] for s in sets], np.uint8)


def pattern_case(n, width, ragged, iupac_rate, seed):
    """(codes, lens, allow, plens): random rows with planted occurrences of random degenerate patterns of lengths
    1, 17, 31 and 32, a poly-A pattern against A runs (overlapping hits), a pattern with a position that allows no
    base, and one site that ends in the last column of a longest row"""
    from multiprime_b200.iupac import allow_masks
    rng = np.random.default_rng(seed)
    codes = SINGLE[rng.integers(0, 4, (n, width))]
    if iupac_rate:
        m = rng.random((n, width)) < iupac_rate
        codes[m] = MULTI[rng.integers(0, len(MULTI), int(m.sum()))]
    lens = np.full(n, width, np.int32)
    if ragged:
        lens = rng.integers(max(40, width // 2), width + 1, n).astype(np.int32)
        lens[rng.integers(0, n)] = width
    pats = []
    for L in (1, 17, 31, 32):
        s = [int(x) for x in SINGLE[rng.integers(0, 4, L)]]
        for j in rng.integers(0, L, int(rng.integers(0, 4))):                  # 2-, 3- and 4-fold positions
            s[j] |= int(rng.integers(1, 16))
        pats.append(s)
    pats.append([1] * 8)                                                        # poly-A
    dead = [int(x) for x in SINGLE[rng.integers(0, 4, 12)]]
    dead[5] = 0                                                                 # a position nothing matches
    pats.append(dead)
    full = int(np.nonzero(lens == width)[0][0])
    taken = np.zeros((n, width), bool)
    taken[full, width - 32:] = True

    def spot(L, r=None, lo=0):
        """a free stretch of L cells (planted sites do not overwrite each other)"""
        for _ in range(50):
            rr = int(rng.integers(0, n)) if r is None else r
            x = int(rng.integers(lo, lens[rr] - L + 1))
            if not taken[rr, x:x + L].any():
                taken[rr, x:x + L] = True
                return rr, x
        return rr, x

    for s in pats:
        L = len(s)
        plant = [spot(L) for _ in range(max(3, n // 8))]
        if width > 65535 + 64:                                                  # around and past column 65535
            plant += [(full, 65535 - L // 2), spot(L, full, 65536)]
        for r, x in plant:
            codes[r, x:x + L] = _expansion(rng, [q if q else 15 for q in s])
            if iupac_rate and rng.random() < 0.3:                               # an IUPAC / N / gap cell inside
                codes[r, x + int(rng.integers(0, L))] = MULTI[rng.integers(0, len(MULTI))]
    for _ in range(max(2, n // 16)):                                            # A runs: overlapping occurrences
        r, x = spot(20)
        codes[r, x:x + 20] = 1
    codes[full, width - 32:] = _expansion(rng, pats[3])                        # a site ending in the last column
    allow = np.array([allow_masks(s) for s in pats], np.uint32)
    plens = np.array([len(s) for s in pats], np.int32)
    return codes, lens, allow, plens


def _upload(backend, ctx, codes, lens):
    from multiprime_b200.core import pack4
    n, width = codes.shape
    junk = codes.copy()                                     # cells past a row's length must never be read
    junk[np.arange(width)[None, :] >= lens[:, None]] = 15
    return backend.Msa(ctx, pack4(junk), n, width, lens=lens)


def _triples(hp, hr, hx):
    return np.stack([np.asarray(hp), np.asarray(hr), np.asarray(hx)], 1).astype(np.int64).reshape(-1, 3)


PATTERN_CASES = [
    pytest.param(1, 300, False, 0.0, id="rows1"),
    pytest.param(31, 300, True, 0.0, id="rows31-ragged"),
    pytest.param(33, 300, False, 0.0, id="rows33"),
    pytest.param(129, 300, True, 0.0, id="rows129-ragged"),
    pytest.param(4999, 300, True, 0.0, id="rows4999-ragged"),
    pytest.param(3, 70_000, True, 0.0, id="wide70000"),
    pytest.param(257, 300, True, 0.03, id="iupac-n-gap-cells"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("n,width,ragged,iupac_rate", PATTERN_CASES)
def test_pattern_hits_equal_plain_search(n, width, ragged, iupac_rate):
    from multiprime_b200 import _lib
    codes, lens, allow, plens = pattern_case(n, width, ragged, iupac_rate, seed=n * 7 + width)
    want = reference_hits(codes, lens, allow, plens)
    ctx = _lib.Context(0)
    msa = _upload(_lib, ctx, codes, lens)
    try:
        got = _triples(*msa.pattern_hits(allow, plens))
    finally:
        msa.close()
        ctx.close()
    assert got.shape == want.shape and (got == want).all()
    per_pat = np.bincount(want[:, 0], minlength=len(plens))
    assert per_pat[-1] == 0 and (per_pat[:-1] > 0).all()            # the dead pattern has none, the others do
    assert (want[:, 2] + plens[want[:, 0]] == width).any()          # a hit ends in the last column
    if width > 65535:
        assert (want[:, 2] > 65535).any()
    if iupac_rate:                  # the case tells the contract apart from "any base of the cell is allowed"
        assert len(reference_hits(codes, lens, allow, plens, exact=False)) > len(want)


@pytest.mark.gpu
def test_pattern_hits_past_default_capacity():
    """a length-1 N pattern hits every single-base cell: more than the 2^20 hits the first call has room for, so the
    call is repeated with the returned count"""
    from multiprime_b200 import _lib
    rng = np.random.default_rng(11)
    n, width = 4001, 300
    codes = SINGLE[rng.integers(0, 4, (n, width))]
    m = rng.random((n, width)) < 0.01
    codes[m] = MULTI[rng.integers(0, len(MULTI), int(m.sum()))]
    lens = np.full(n, width, np.int32)
    allow = np.array([[1, 1, 1, 1], [1, 0, 0, 0]], np.uint32)
    plens = np.array([1, 1], np.int32)
    want = reference_hits(codes, lens, allow, plens)
    assert len(want) > (1 << 20)
    ctx = _lib.Context(0)
    msa = _upload(_lib, ctx, codes, lens)
    try:
        got = _triples(*msa.pattern_hits(allow, plens))
    finally:
        msa.close()
        ctx.close()
    assert got.shape == want.shape and (got == want).all()


@pytest.mark.gpu
def test_upload_column_limit():
    """65535 words of 32 columns (2097120) upload and are searched to the last column; one more column is refused with
    a message that names the limit"""
    from multiprime_b200 import _lib
    from multiprime_b200.core import pack4
    width = 65535 * 32
    codes = np.ones((1, width + 1), np.uint8)                       # one poly-A line
    ctx = _lib.Context(0)
    try:
        msa = _lib.Msa(ctx, pack4(codes[:, :width]), 1, width)
        got = _triples(*msa.pattern_hits(np.array([[7, 0, 0, 0]], np.uint32), np.array([3], np.int32)))
        msa.close()
        assert len(got) == width - 2 and got[-1, 2] == width - 3
        with pytest.raises(_lib.MpbError, match="2097120 columns"):
            _lib.Msa(ctx, pack4(codes), 1, width + 1)
    finally:
        ctx.close()


def test_fake_device_pattern_hits_follow_the_contract():
    """the CPU double of mpb_pattern_hits and the plain search agree (IUPAC cells, ragged rows)"""
    from tests import fake_device
    codes, lens, allow, plens = pattern_case(29, 120, True, 0.05, seed=3)
    msa = _upload(fake_device, fake_device.Context(), codes, lens)
    got = _triples(*msa.pattern_hits(allow, plens))
    want = reference_hits(codes, lens, allow, plens)
    assert got.shape == want.shape and (got == want).all()
    assert len(want) > 20


# ---------------------------------------------------------------------------------------------------------------
# pair coverage
# ---------------------------------------------------------------------------------------------------------------
def _popcount_table(a, b):
    """t[x, y] = popcount(a[x] | b[y]) over the word axis"""
    t = np.zeros((len(a), len(b)), np.int64)
    for x in range(len(a)):
        t[x] = np.bitwise_count(a[x][None, :] | b).sum(1)
    return t


def _bit_rows(rng, shape):
    """random words; row r keeps each bit with probability 2^-(r % 4); row 0 is empty, row 1 full"""
    out = rng.integers(0, 1 << 32, shape, dtype=np.uint64).astype(np.uint32)
    for r in range(shape[0]):
        for _ in range(r % 4):
            out[r] &= rng.integers(0, 1 << 32, shape[1:], dtype=np.uint64).astype(np.uint32)
    out[0], out[1] = 0, 0xFFFFFFFF
    return out


def _pairs(rng, rows, n_pairs):
    pf = rng.integers(0, rows, n_pairs).astype(np.int32)
    pr = rng.integers(0, rows, n_pairs).astype(np.int32)
    pr[::7] = pf[::7]                                               # the same primer on both sides
    pf[-1], pr[-1] = rows - 1, rows - 1
    return pf, pr


def _dev_copy(ctx, host):
    from multiprime_b200 import _lib
    buf = _lib.DevBuf(ctx, host.shape, host.dtype)
    _lib.check(_lib.load().mpb_ctx_memcpy(ctx.h, C.c_void_p(buf.p), _lib.ptr(host), host.nbytes))
    return buf


@pytest.mark.gpu
@pytest.mark.parametrize("words", [1, 2, 31, 32, 33, 129, 31_251])
def test_pair_cover_equals_numpy(words):
    """words = 31251 holds 10^6 + 7 sequences; rows are few, so numpy evaluates every (pf, pr) combination once"""
    from multiprime_b200 import _lib
    rng = np.random.default_rng(words)
    rows = 24
    uf, ur = _bit_rows(rng, (rows, words)), _bit_rows(rng, (rows, words))
    b3 = _bit_rows(rng, (rows, 3, words))
    pf, pr = _pairs(rng, rows, 100_003)
    ctx = _lib.Context(0)
    try:
        want = _popcount_table(uf, ur)[pf, pr]
        assert (ctx.pair_cover(uf, ur, pf, pr) == want).all()
        want3 = _popcount_table(b3[:, 0] | b3[:, 2], b3[:, 1] | b3[:, 2])[pf, pr]
        assert (ctx.pair_cover3(b3, pf, pr) == want3).all()
        dev = _dev_copy(ctx, b3)
        assert (ctx.pair_cover3(dev, pf, pr) == want3).all()
        dev.close()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_scan_bit_vectors_have_no_padding_bits():
    """Hist.cscan bit vectors of an alignment whose row count is not a multiple of 32 (gap-rich, ragged rows, IUPAC
    cells): no bit at or past n_seq in any of the three vectors, the device copy equals the host one, and
    pair_cover3 on the device buffer equals numpy on its host copy"""
    from multiprime_b200 import _lib, core, synth
    from tests.test_gpu_colscan import _random_candidates
    n, L, k, v = 1037, 220, 20, 2
    rng = np.random.default_rng(1037)
    codes = synth.synth_codes(n, L, seed=9, gap_rate=0.08, iupac_rate=0.01, term_gap=0.5)
    lens = rng.integers(L // 2, L + 1, n).astype(np.int32)
    for s, m in enumerate(lens):
        codes[s, m:] = 0
    pos = sorted(set(rng.integers(0, L // 2 - k, 12).tolist()))
    wins, allows, trials = _random_candidates(rng, codes, pos, k)
    cands = _lib.make_cands(wins, allows, trials)
    slots = np.arange(len(cands), dtype=np.int32)
    fmask, rmask = core.strict_masks("1,2,-1", k)
    ctx = _lib.Context(0)
    msa = _lib.Msa(ctx, core.pack4(codes), n, L, lens=lens)
    try:
        with msa.hist(k, v, pos) as h:
            counts, host = h.cscan(fmask, rmask, cands, bits_slot=slots)
            counts_d, dev = h.cscan(fmask, rmask, cands, bits_slot=slots, bits_out="device")
        words = (n + 31) // 32
        assert host.shape == (len(cands), 3, words)
        pad = ~np.uint32((1 << (n % 32)) - 1)
        assert not (host[:, :, -1] & pad).any()
        assert (dev.to_host() == host).all() and (counts_d == counts).all()
        assert host[:, 2].any() and host[:, 0].any()                   # gap rows and non-cover rows do occur
        pf, pr = _pairs(rng, len(cands), 20_000)
        want = _popcount_table(host[:, 0] | host[:, 2], host[:, 1] | host[:, 2])[pf, pr]
        assert (ctx.pair_cover3(dev, pf, pr) == want).all()
        assert want.max() <= n
        dev.close()
    finally:
        msa.close()
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------
# dimer grid
# ---------------------------------------------------------------------------------------------------------------
_RC = str.maketrans("ACGT", "TGCA")


def dimer_primers(n, seed):
    """seeded random primers of lengths 5..32: mostly ACGT with 0 to 4 degenerate codes, some with N in the last five
    bases, duplicates, and planted reverse complements of other primers' 3' ends (hits at d2 = 0 and further in)"""
    from multiprime_b200.iupac import BASES, CHAR_CODE, ORDER
    rng = np.random.default_rng(seed)
    dege = "RYMKSWHBVD"
    out = []
    while len(out) < n:
        r = rng.random()
        if out and r < 0.04:                                                     # duplicate
            out.append(out[int(rng.integers(0, len(out)))])
            continue
        L = int(rng.choice([5, 6, 12, 18, 20, 25, 32]))
        s = list(rng.choice(list("ACGT"), L))
        for j in rng.integers(0, L, int(rng.integers(0, 5))):
            s[j] = dege[int(rng.integers(0, len(dege)))]
        if rng.random() < 0.08:                                                  # N in the last five bases
            for j in rng.integers(max(0, L - 5), L, int(rng.integers(1, 3))):
                s[j] = "N"
        if out and L >= 8 and r > 0.75:                                          # a partner's 3' end, reverse-complemented
            other = out[int(rng.integers(0, len(out)))]
            e = "".join(BASES[ORDER[CHAR_CODE[ch]][0]] for ch in other[-int(rng.integers(5, min(len(other), L) + 1)):])
            t = e.translate(_RC)[::-1]
            at = L - len(t) if rng.random() < 0.5 else int(rng.integers(0, L - len(t) + 1))
            s[at:at + len(t)] = list(t)
        out.append("".join(s))
    return out


def _engine(ctx, primers):
    from multiprime_b200 import _lib
    from multiprime_b200.dimer import dg_consts, loss_table
    from multiprime_b200.iupac import sets_of
    return _lib.Dimer(ctx, [sets_of(p) for p in primers], 5, 18, True, loss_table(3.96), dg_consts())


@pytest.mark.gpu
def test_dimer_prefilter_keeps_every_dimer():
    """grid over all rows == the pairs with a first hit when k_dimer_pairs runs on every (i, j >= i) pair"""
    from multiprime_b200 import _lib
    primers = dimer_primers(2500, seed=2500)
    n = len(primers)
    ctx = _lib.Context(0)
    eng = _engine(ctx, primers)
    try:
        hi, hj, ho, hd, nt = eng.grid(0, n)
        pi, pj = np.triu_indices(n)
        fh, d2 = eng.pairs(pi.astype(np.int32), pj.astype(np.int32))
        # the wide-block (few pairs) and narrow-block launches agree: 64 pairs per call is below 4 x SMs
        sub = np.concatenate([np.nonzero(fh >= 0)[0][:3000], np.arange(0, len(pi), 997)])
        parts = [eng.pairs(pi[sub[a:a + 64]].astype(np.int32), pj[sub[a:a + 64]].astype(np.int32))
                 for a in range(0, len(sub), 64)]
    finally:
        eng.close()
        ctx.close()
    got = sorted(zip(hi.tolist(), hj.tolist(), ho.tolist(), hd.tolist()))
    keep = fh >= 0
    want = sorted(zip(pi[keep].tolist(), pj[keep].tolist(), fh[keep].tolist(), d2[keep].tolist()))
    assert got == want
    assert nt >= len(got) and nt < len(pi)                            # the prefilter does drop pairs
    assert (d2[keep] == 0).any() and (d2[keep] > 0).any()
    assert (np.concatenate([p[0] for p in parts]) == fh[sub]).all()
    assert (np.concatenate([p[1] for p in parts]) == d2[sub]).all()


def _findimer(tmp_path, primers):
    from multiprime_b200 import findimer
    fa = tmp_path / "p.fa"
    fa.write_text("".join(">P%04d\n%s\n" % (i, p) for i, p in enumerate(primers)))
    return findimer.Dimer(primer_file=str(fa), outfile=str(tmp_path / "o.txt"), threshold=3.96, nproc=1)


@pytest.mark.gpu
def test_findimer_rows_do_not_depend_on_the_band(tmp_path):
    app = _findimer(tmp_path, dimer_primers(2500, seed=77))
    rows = [app.find(rows_per_band=b) for b in (1, 7, 64, len(app.primers_list))]
    assert len(rows[0]) > 1000
    for r in rows[1:]:
        assert r == rows[0]


@pytest.mark.gpu
def test_findimer_equals_dimer_oracle(tmp_path):
    """300 primers: the drop-in's rows equal oracle.dimer_oracle.find_dimers (pinned to finDimer_V4)"""
    from oracle import dimer_oracle
    primers = dimer_primers(2500, seed=77)[:300]
    app = _findimer(tmp_path, primers)
    rows = app.find()
    want = dimer_oracle.find_dimers(app.primers, 3.96)
    assert len(want) > 50
    assert [tuple(r) for r in rows] == [tuple(r) for r in want]
