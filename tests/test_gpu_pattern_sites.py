"""mpb_pattern_sites (the search behind primer_coverage) against a plain numpy statement of the mismatch rule, against
mpb_pattern_hits at v = 0, and against the core's own per-sequence verdict (Msa.scan's non-cover bits) for window
primers; the CPU double follows the same contract."""
import numpy as np
import pytest

from tests.test_gpu_tool_kernels import MULTI, SINGLE, _expansion, _triples, pattern_case


def reference_sites(codes, lens, allow, plens, strict, v):
    """every (pattern, row, position, mismatches) with the site inside lens[row], at most v cells that are not exactly
    one allowed base, none of them at a strict position -> int64[n, 4] sorted"""
    n, width = codes.shape
    single = np.zeros(16, bool)
    single[SINGLE] = True
    out = []
    for p, L in enumerate(plens):
        L = int(L)
        nx = width - L + 1
        if nx <= 0:
            continue
        mis = np.zeros((n, nx), np.int64)
        dead = np.zeros((n, nx), bool)
        for i in range(L):
            allowed = sum(((int(allow[p][q]) >> i) & 1) << q for q in range(4))
            ok = ((np.arange(16) & allowed) != 0) & single
            m = ~ok[codes[:, i:i + nx]]
            mis += m
            if (int(strict[p]) >> i) & 1:
                dead |= m
        good = (mis <= v) & ~dead & (np.arange(nx)[None, :] + L <= np.asarray(lens)[:, None])
        r, x = np.nonzero(good)
        out.append(np.stack([np.full(len(r), p), r, x, mis[r, x]], 1))
    return np.concatenate(out).astype(np.int64) if out else np.zeros((0, 4), np.int64)


def sites_case(n, width, ragged, iupac_rate, v, seed):
    """random rows with junk bases past each row's length, and planted sites of random degenerate patterns with random
    strict positions: with exactly 0, v and v + 1 mismatches, with a mismatch on a strict position, with IUPAC / N / gap
    cells inside, and hanging past a row's end by 1..v cells whose junk matches the pattern"""
    rng = np.random.default_rng(seed)
    codes = SINGLE[rng.integers(0, 4, (n, width))]
    if iupac_rate:
        m = rng.random((n, width)) < iupac_rate
        codes[m] = MULTI[rng.integers(0, len(MULTI), int(m.sum()))]
    lens = np.full(n, width, np.int32)
    if ragged:
        lens = rng.integers(max(40, width // 2), width + 1, n).astype(np.int32)
    pats, strict = [], []
    for L in (20, 24, 31, 32):
        s = [int(x) for x in SINGLE[rng.integers(0, 4, L)]]
        for j in rng.integers(0, L, int(rng.integers(0, 4))):
            s[j] |= int(rng.integers(1, 16))
        pats.append(s)
        strict.append(int(sum(1 << int(j) for j in rng.choice(L, 3, replace=False))) if L != 24 else 0)
    for p, s in enumerate(pats):
        L = len(s)
        free = [i for i in range(L) if not (strict[p] >> i) & 1]
        for _ in range(max(4, n // 8)):
            r = int(rng.integers(0, n))
            x = int(rng.integers(0, lens[r] - L + 1))
            site = _expansion(rng, s)
            k = int(rng.choice([0, v, v + 1]))
            for i in rng.choice(free, min(k, len(free)), replace=False):
                site[i] = MULTI[rng.integers(0, len(MULTI))] if rng.random() < 0.5 else \
                    SINGLE[[q for q in range(4) if not (s[i] >> q) & 1][0]] if s[i] != 15 else 0
            if strict[p] and rng.random() < 0.25:                        # a mismatch on a strict position
                site[int(np.flatnonzero([(strict[p] >> i) & 1 for i in range(L)])[0])] = 0
            codes[r, x:x + L] = site
        for j in range(1, v + 1):                                         # hanging past the row end by j cells
            r = int(rng.integers(0, n))
            x = int(lens[r]) - L + j
            if x >= 0 and x + L <= width:
                codes[r, x:x + L] = _expansion(rng, s)
    allow = np.array([[sum(((c >> b) & 1) << i for i, c in enumerate(s)) for b in range(4)] for s in pats], np.uint32)
    plens = np.array([len(s) for s in pats], np.int32)
    return codes, lens, allow, plens, np.array(strict, np.uint32)


def _upload(backend, ctx, codes, lens):
    from multiprime_b200.core import pack4
    return backend.Msa(ctx, pack4(codes), codes.shape[0], codes.shape[1], lens=lens)


SITE_CASES = [
    pytest.param(1, 300, False, 0.0, 1, id="rows1-v1"),
    pytest.param(33, 300, True, 0.03, 3, id="rows33-ragged-iupac-v3"),
    pytest.param(4999, 300, True, 0.0, 1, id="rows4999-ragged-v1"),
    pytest.param(257, 300, True, 0.03, 0, id="rows257-iupac-v0"),
    pytest.param(33, 300, False, 0.0, 15, id="rows33-v15"),
    pytest.param(129, 300, True, 0.02, 15, id="rows129-ragged-iupac-v15"),
    pytest.param(3, 70_000, True, 0.0, 3, id="wide70000-v3"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("n,width,ragged,iupac_rate,v", SITE_CASES)
def test_pattern_sites_equal_plain_rule(n, width, ragged, iupac_rate, v):
    from multiprime_b200 import _lib
    codes, lens, allow, plens, strict = sites_case(n, width, ragged, iupac_rate, v, seed=n * 13 + v)
    want = reference_sites(codes, lens, allow, plens, strict, v)
    ctx = _lib.Context(0)
    msa = _upload(_lib, ctx, codes, lens)
    try:
        got = np.stack(msa.pattern_sites(allow, plens, strict, v), 1).astype(np.int64).reshape(-1, 4)
    finally:
        msa.close()
        ctx.close()
    assert got.shape == want.shape and (got == want).all()
    assert len(want) and (want[:, 3] == v).any()
    if ragged and v:                  # junk past the row ends would add sites if lens were not checked
        loose = reference_sites(codes, np.full(n, width, np.int32), allow, plens, strict, v)
        assert len(loose) > len(want)


@pytest.mark.gpu
def test_pattern_sites_past_default_capacity():
    """a 16-base pattern with 15 mismatches allowed binds almost everywhere: more sites than the first call has room
    for, so the call is repeated with the returned count"""
    from multiprime_b200 import _lib
    rng = np.random.default_rng(4)
    n, width = 4001, 300
    codes = SINGLE[rng.integers(0, 4, (n, width))]
    lens = np.full(n, width, np.int32)
    allow = np.array([[0xFFFF, 0, 0, 0]], np.uint32)
    plens, strict = np.array([16], np.int32), np.array([0], np.uint32)
    want = reference_sites(codes, lens, allow, plens, strict, 15)
    assert len(want) > (1 << 20)
    ctx = _lib.Context(0)
    msa = _upload(_lib, ctx, codes, lens)
    try:
        got = np.stack(msa.pattern_sites(allow, plens, strict, 15), 1).astype(np.int64)
    finally:
        msa.close()
        ctx.close()
    assert got.shape == want.shape and (got == want).all()


@pytest.mark.gpu
@pytest.mark.parametrize("n,width,ragged,iupac_rate", [(33, 300, False, 0.0), (129, 300, True, 0.0),
                                                       (257, 300, True, 0.03)])
def test_pattern_sites_v0_equal_pattern_hits(n, width, ragged, iupac_rate):
    from multiprime_b200 import _lib
    codes, lens, allow, plens = pattern_case(n, width, ragged, iupac_rate, seed=n * 7 + width)
    ctx = _lib.Context(0)
    msa = _upload(_lib, ctx, codes, lens)
    try:
        hits = _triples(*msa.pattern_hits(allow, plens))
        hp, hr, hx, hm = msa.pattern_sites(allow, plens, np.zeros(len(plens), np.uint32), 0)
    finally:
        msa.close()
        ctx.close()
    assert (np.asarray(hm) == 0).all()
    assert len(hits) and (_triples(hp, hr, hx) == hits).all() and len(hp) == len(hits)


@pytest.mark.gpu
def test_pattern_sites_refuse_bad_bounds():
    from multiprime_b200 import _lib
    codes = SINGLE[np.zeros((1, 64), np.int64)]
    ctx = _lib.Context(0)
    msa = _upload(_lib, ctx, codes, np.array([64], np.int32))
    try:
        allow, strict = np.array([[0xFF, 0, 0, 0]], np.uint32), np.zeros(1, np.uint32)
        with pytest.raises(_lib.MpbError, match="match everywhere"):
            msa.pattern_sites(allow, np.array([8], np.int32), strict, 8)
        with pytest.raises(_lib.MpbError, match="at most 15"):
            msa.pattern_sites(np.array([[0xFFFFFFFF, 0, 0, 0]], np.uint32), np.array([32], np.int32), strict, 16)
    finally:
        msa.close()
        ctx.close()


def test_cpu_double_pattern_sites_follow_the_contract():
    from tests import fake_pattern_sites
    for v in (0, 3):
        codes, lens, allow, plens, strict = sites_case(29, 120, True, 0.05, v, seed=3 + v)
        msa = _upload(fake_pattern_sites, fake_pattern_sites.Context(), codes, lens)
        got = np.stack(msa.pattern_sites(allow, plens, strict, v), 1).astype(np.int64).reshape(-1, 4)
        want = reference_sites(codes, lens, allow, plens, strict, v)
        assert got.shape == want.shape and (got == want).all() and len(want) > 5


# ---------------------------------------------------------------------------------------------------------------
# the core's verdict: a window primer scored by mis_primer_check binds exactly the sequences the scan covers
# ---------------------------------------------------------------------------------------------------------------
def _core_cross_check(backend):
    from multiprime_b200.core import strict_masks
    from multiprime_b200.iupac import allow_masks
    rng = np.random.default_rng(8)
    n, width, k, v = 300, 90, 18, 2
    root = rng.integers(0, 4, width)
    base = np.where(rng.random((n, width)) < 0.06, rng.integers(0, 4, (n, width)), root[None, :])
    codes = SINGLE[base]
    fmask, rmask = strict_masks("1,2,-1", k)
    ctx = backend.Context(0)
    msa = _upload(backend, ctx, codes, np.full(n, width, np.int32))
    checked = 0
    try:
        for p in (3, 40, 71):
            sets = [int(SINGLE[b]) for b in root[p:p + k]]
            for j in rng.choice(k, 2, replace=False):
                sets[j] |= int(SINGLE[rng.integers(0, 4)])
            allow = np.array([allow_masks(sets)], np.uint32)
            _, bits = msa.scan(k, v, fmask, rmask, [p], allow, bits_slot=[0])
            for j, mask in ((0, fmask), (1, rmask)):
                hp, hr, hx, _ = msa.pattern_sites(allow, np.array([k], np.int32), np.array([mask], np.uint32), v)
                bound = set(np.asarray(hr)[np.asarray(hx) == p].tolist())
                covered = {s for s in range(n) if not (int(bits[0, j, s >> 5]) >> (s & 31)) & 1}
                assert bound == covered, (p, j)
                assert 0 < len(covered) < n
                checked += 1
    finally:
        msa.close()
        ctx.close()
    assert checked == 6


@pytest.mark.gpu
def test_pattern_sites_agree_with_core_scan():
    from multiprime_b200 import _lib
    _core_cross_check(_lib)


def test_cpu_double_pattern_sites_agree_with_core_scan():
    from tests import fake_pattern_sites
    _core_cross_check(fake_pattern_sites)
