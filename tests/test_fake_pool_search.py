"""The CPU double of mpb_pool_search (tests/fake_pool_search.py) pinned on its own: it finds the brute-force optimum of
tiny instances, keeps the pools balanced at every step, reports costs that match its assignments, and solves planted
instances."""
import itertools

import numpy as np
import pytest

from tests import fake_pool_search as fps


def random_w(n, density, rng, top=12):
    w = np.triu(rng.integers(1, top + 1, (n, n)) * (rng.random((n, n)) < density), 1)
    return (w + w.T).astype(np.uint8)


def planted_w(n, P, rng, density=0.3, top=12):
    """conflicts only between pairs of different pools of a hidden balanced partition"""
    hidden = rng.permutation(np.arange(n) % P)
    w = random_w(n, density, rng, top)
    w[hidden[:, None] == hidden[None, :]] = 0
    return w


def cost_of(w, pool):
    same = pool[:, None] == pool[None, :]
    return int((w.astype(np.int64) * same).sum()) // 2


def brute_force(w, P):
    n = len(w)
    sizes = sorted([n // P + (p < n % P) for p in range(P)])
    best = None
    for pool in itertools.product(range(P), repeat=n):
        if sorted(np.bincount(pool, minlength=P).tolist()) != sizes:
            continue
        c = cost_of(w, np.array(pool))
        best = c if best is None else min(best, c)
    return best


@pytest.mark.parametrize("P", [2, 3])
@pytest.mark.parametrize("n", [4, 7, 10])
@pytest.mark.parametrize("density", [0.3, 0.8])
def test_brute_force_optimum(n, P, density):
    rng = np.random.default_rng(n * 100 + P * 10 + int(density * 10))
    w = random_w(n, density, rng)
    res = fps.pool_search(w, P, 7, 0, 16, 300)
    assert int(res["cost"].min()) == brute_force(w, P)


@pytest.mark.parametrize("n,P", [(10, 3), (33, 8), (64, 7), (31, 2)])
def test_every_step_is_balanced_and_costs_match(n, P):
    rng = np.random.default_rng(n + P)
    w = random_w(n, 0.4, rng)
    sizes = sorted([n // P + (p < n % P) for p in range(P)])
    seen = []

    def trace(t, pool, cost):
        assert sorted(np.bincount(pool, minlength=P).tolist()) == sizes
        assert cost == cost_of(w, pool)
        seen.append(cost)

    best, step, assign = fps.restart_search(w, P, 3, 1, 200, trace)
    assert len(seen) > 1
    assert best == min(seen) == seen[step] == cost_of(w, assign)
    assert seen.index(best) == step


@pytest.mark.parametrize("n,P", [(40, 2), (64, 8), (33, 3)])
def test_planted_instances_reach_zero(n, P):
    rng = np.random.default_rng(n * P)
    w = planted_w(n, P, rng)
    res = fps.pool_search(w, P, 1, 0, 4, 2000)
    assert int(res["cost"].min()) == 0
    for c, a in zip(res["cost"], res["assign"]):
        assert c == cost_of(w, a.astype(np.int64))


def test_refusals():
    w = np.zeros((4, 4), np.uint8)
    for args, msg in (((w, 0, 0, 1, 1), "pools"), ((w, 33, 0, 1, 1), "pools"), ((w, 5, 0, 1, 1), "pools <= pairs"),
                      ((np.zeros((513, 513), np.uint8), 2, 0, 1, 1), "pairs"), ((w, 2, 2, 1, 1), "restarts"),
                      ((w, 2, 0, 1, 1 << 20), "iterations")):
        with pytest.raises(fps.MpbError, match=msg):
            fps.pool_search(args[0], args[1], 1, args[2], args[3], args[4])
    bad = w.copy()
    bad[0, 1] = 1
    with pytest.raises(fps.MpbError, match="symmetric"):
        fps.pool_search(bad, 2, 1, 0, 1, 1)
    bad = w.copy()
    bad[2, 2] = 1
    with pytest.raises(fps.MpbError, match="diagonal"):
        fps.pool_search(bad, 2, 1, 0, 1, 1)
