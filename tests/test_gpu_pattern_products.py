"""mpb_pattern_products against its CPU double (tests/fake_pattern_products.py, itself pinned to a plain restatement by
tests/test_primer_specificity.py): every output, for several mismatch bounds, row strides, listed-flag tables and chunk
budgets, on a case with runs of one (primer, record) longer than a join block; and the packing limits it refuses."""
import numpy as np
import pytest

from tests.test_primer_coverage import IUPAC, rc
from tests.test_primer_specificity import make_spec_case

pytestmark = pytest.mark.gpu


def _inputs(tmp_path, seed, stride):
    """(rows, width, panel, primers, record offsets, lengths, lo, hi) of the specificity case plus a record of 300
    inverted F / R repeats: one (primer, record) run of about 600 left sites"""
    from multiprime_b200 import primer_coverage as pc
    from multiprime_b200 import primer_specificity as ps
    from multiprime_b200.pcr_product import parse_primers
    fa, pf, lo, hi = make_spec_case(tmp_path, seed)
    pairs = parse_primers(pf, "fa")
    f, r = (("".join(IUPAC[ch][0] for ch in p)) for p in list(pairs.values())[0])
    rng = np.random.default_rng(seed)
    unit = lambda: f + "".join(rng.choice(list("ACGT"), 25)) + rc(f) + r + "".join(rng.choice(list("ACGT"), 9))  # noqa
    with open(fa, "a") as fh:
        fh.write(">repeats\n%s\n" % "".join(unit() for _ in range(300)))
    old = pc.S
    pc.S = stride
    try:
        t = pc.read_targets(fa)
        panel = pc.Panel(pairs, "1,2,-1")
        rows, width, starts = pc.layout(t, panel.lmax)
    finally:
        pc.S = old
    return rows, width, panel, ps.Primers(panel), starts, t.lens, lo, hi


def _call(backend, rows, width, panel, primers, starts, lens, lo, hi, v, stride, listed, max_rows, chunk):
    ctx = backend.Context.shared(0) if backend.__name__.endswith("_lib") else None
    msa = backend.Msa(ctx, rows, len(rows), width, row_bytes=rows.shape[1])
    try:
        return msa.pattern_products(panel.allow, panel.plen, panel.strict, v, primers.pat_primer, primers.pat_side,
                                    len(primers.seqs), stride, starts, lens, lo, hi, listed, max_rows, chunk)
    finally:
        msa.close()


@pytest.mark.parametrize("stride", [64, 4096])
@pytest.mark.parametrize("v", [0, 1, 3])
def test_entry_point_matches_double(tmp_path, stride, v):
    from multiprime_b200 import _lib
    from tests import fake_pattern_products
    rows, width, panel, primers, starts, lens, lo, hi = _inputs(tmp_path, v, stride)
    n = len(primers.seqs)
    rng = np.random.default_rng(v)
    for listed, max_rows in ((primers.listed, 1 << 20), (np.ones((n, n), np.uint8), 1 << 20),
                             ((rng.random((n, n)) < 0.5).astype(np.uint8), 17), (primers.listed, 0)):
        want = _call(fake_pattern_products, rows, width, panel, primers, starts, lens, lo, hi, v, stride, listed,
                     max_rows, 0)
        assert max(want["comb"][:, :, 1].max(), 0) > 0
        for chunk in (0, 1, 3, 130):
            got = _call(_lib, rows, width, panel, primers, starts, lens, lo, hi, v, stride, listed, max_rows, chunk)
            for k in ("comb", "union", "rows", "stats"):
                np.testing.assert_array_equal(got[k], want[k], err_msg="%s chunk %d" % (k, chunk))
            assert got["n_listed"] == want["n_listed"]
    every = _call(fake_pattern_products, rows, width, panel, primers, starts, lens, lo, hi, v, stride,
                  np.ones((n, n), np.uint8), 1 << 20, 0)["rows"]
    assert (every[every[:, 0] == len(lens) - 1, 7] > 128).any()   # a group of the repeats spans several join blocks


def test_packing_limits_are_refused(tmp_path):
    from multiprime_b200 import _lib
    rows, width, panel, primers, starts, lens, lo, hi = _inputs(tmp_path, 1, 64)
    args = (rows, width, panel, primers, starts, lens)
    with pytest.raises(_lib.MpbError, match="lo <= hi <= 8388607"):
        _call(_lib, *args, 50, 1 << 23, 1, 64, primers.listed, 10, 0)
    big = np.array(lens, np.int64)
    big[-1] = 1 << 32
    with pytest.raises(_lib.MpbError, match="packed product start"):
        _call(_lib, rows, width, panel, primers, starts, big, lo, hi, 1, 64, primers.listed, 10, 0)
