"""mpb_pool_search against its CPU double (tests/fake_pool_search.py), restart by restart: best cost, best step and the
assignment at that step, over pair counts, pool counts, weight shapes and step budgets; restarts split over calls; every
refusal; and the tool's default budget on a planted 512-pair, 8-pool instance."""
import numpy as np
import pytest

from multiprime_b200 import primer_pools as pp
from tests import fake_pool_search as fps
from tests.test_fake_pool_search import cost_of, planted_w, random_w

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1), (2, 1), (2, 2), (31, 2), (31, 7), (33, 3), (33, 32), (64, 8), (64, 7), (200, 3), (200, 8),
          (512, 2), (512, 7), (512, 32)]
KINDS = ["zero", "full", "sparse", "dense", "planted"]


def make_w(kind, n, P, seed):
    rng = np.random.default_rng(seed)
    if kind == "zero":
        return np.zeros((n, n), np.uint8)
    if kind == "full":
        w = np.full((n, n), 12, np.uint8)
        np.fill_diagonal(w, 0)
        return w
    if kind == "sparse":
        return random_w(n, 3.0 / max(n, 1), rng)
    if kind == "dense":
        return random_w(n, 0.6, rng)
    return planted_w(n, P, rng)


@pytest.fixture(scope="module")
def ctx():
    from multiprime_b200 import _lib
    return _lib.Context(0)


def _compare(ctx, w, P, seed, r0, r1, iters):
    got = ctx.pool_search(w, P, seed, r0, r1, iters)
    want = fps.pool_search(w, P, seed, r0, r1, iters)
    for k in ("cost", "step", "assign"):
        assert np.array_equal(got[k], want[k]), (k, got[k], want[k])
    for c, a in zip(got["cost"], got["assign"]):
        assert c == cost_of(w, a.astype(np.int64))
    return got


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n,P", SHAPES)
def test_matches_double(ctx, n, P, kind):
    w = make_w(kind, n, P, n * 37 + P)
    iters = 2000 if n <= 64 else 400 if n <= 200 else 120
    _compare(ctx, w, P, n + P, 0, 3 if n < 512 else 2, iters)


@pytest.mark.parametrize("iters", [0, 1])
@pytest.mark.parametrize("n,P", SHAPES)
def test_zero_and_one_step(ctx, n, P, iters):
    w = make_w("dense", n, P, n + 5)
    got = _compare(ctx, w, P, 11, 5, 9, iters)
    if iters == 0:
        assert (got["step"] == 0).all()


def test_long_budget(ctx):
    """a few thousand steps on an instance the search does not solve: tabu tenure, aspiration and stalls all occur"""
    w = make_w("dense", 64, 3, 99)
    got = _compare(ctx, w, 3, 5, 0, 2, 4000)
    assert (got["cost"] > 0).all()


@pytest.mark.parametrize("n,P", [(33, 8), (200, 3)])
def test_split_restarts_equal_one_call(ctx, n, P):
    w = make_w("dense", n, P, 3)
    one = ctx.pool_search(w, P, 42, 0, 9, 300)
    parts = [ctx.pool_search(w, P, 42, a, b, 300) for a, b in ((0, 2), (2, 3), (3, 3), (3, 9))]
    for k in ("cost", "step", "assign"):
        assert np.array_equal(one[k], np.concatenate([p[k] for p in parts])), k
    assert np.array_equal(ctx.pool_search(w, P, 42, 4, 6, 300)["assign"], one["assign"][4:6])


def test_refusals(ctx):
    from multiprime_b200._lib import MpbError
    w = np.zeros((4, 4), np.uint8)
    cases = [((w, 0, 0, 1, 1), "1 <= pools <= 32"), ((w, 33, 0, 1, 1), "1 <= pools <= 32"),
             ((w, 5, 0, 1, 1), "need pools <= pairs"), ((np.zeros((513, 513), np.uint8), 2, 0, 1, 1), "pairs <= 512"),
             ((np.zeros((0, 0), np.uint8), 1, 0, 1, 1), "pairs <= 512"), ((w, 2, 2, 1, 1), "0 <= r0 <= r1"),
             ((w, 2, -1, 1, 1), "0 <= r0 <= r1"), ((w, 2, 0, (1 << 24) + 1, 1), "0 <= r0 <= r1"),
             ((w, 2, 0, 1, 1 << 20), "iterations <= 1048575"), ((w, 2, 0, 1, -1), "iterations <= 1048575")]
    for (ww, P, r0, r1, it), msg in cases:
        with pytest.raises(MpbError, match=msg) as e:
            ctx.pool_search(ww, P, 1, r0, r1, it)
        assert e.value.code == -1
    bad = w.copy()
    bad[0, 1] = 1
    with pytest.raises(MpbError, match="not symmetric"):
        ctx.pool_search(bad, 2, 1, 0, 1, 1)
    bad = w.copy()
    bad[2, 2] = 3
    with pytest.raises(MpbError, match="diagonal must be zero"):
        ctx.pool_search(bad, 2, 1, 0, 1, 1)


def test_defaults_solve_planted_512_in_8_pools(ctx):
    w = planted_w(512, 8, np.random.default_rng(2024), density=0.05)
    res = ctx.pool_search(w, 8, pp.SEED, 0, pp.RESTARTS, pp.ITERATIONS)
    assert int(res["cost"].min()) == 0
    k = int(np.argmin(res["cost"]))
    assert cost_of(w, res["assign"][k].astype(np.int64)) == 0
