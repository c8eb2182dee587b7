"""The CPU double of mpb_pool_search: the search rule of multiprime_b200/primer_pools.py stated directly, numpy within
a step.

TEST INFRASTRUCTURE ONLY: pass this module as the backend of multiprime_b200.primer_pools to run the tool's host logic
without a GPU (its Msa is tests/fake_pattern_products.py's, its Dimer tests/fake_device.py's);
tests/test_gpu_pool_search.py pins the real entry point to restart_search restart by restart."""
from __future__ import annotations

import numpy as np

from multiprime_b200._lib import MpbError
from multiprime_b200.primer_pools import search_hash
from tests.fake_device import Dimer  # noqa: F401  (the backend's Dimer)
from tests.fake_pattern_products import Context as _Context
from tests.fake_pattern_products import Msa  # noqa: F401  (the backend's Msa)

BIAS = 1 << 24


def check_args(w, n_pools, r0, r1, iterations):
    """mpb_pool_search's refusals"""
    n = w.shape[0]
    if not 1 <= n <= 512:
        raise MpbError(-1, "%d pairs: need 1 <= pairs <= 512" % n)
    if not 1 <= n_pools <= 32:
        raise MpbError(-1, "%d pools: need 1 <= pools <= 32" % n_pools)
    if n_pools > n:
        raise MpbError(-1, "%d pools for %d pairs: need pools <= pairs" % (n_pools, n))
    if not 0 <= r0 <= r1 <= 1 << 24:
        raise MpbError(-1, "restarts [%d, %d): need 0 <= r0 <= r1 <= %d" % (r0, r1, 1 << 24))
    if not 0 <= iterations <= (1 << 20) - 1:
        raise MpbError(-1, "%d iterations: need 0 <= iterations <= %d" % (iterations, (1 << 20) - 1))
    if np.diagonal(w).any():
        raise MpbError(-1, "the diagonal must be zero")
    if (w != w.T).any():
        raise MpbError(-1, "w is not symmetric")


def restart_search(w, P: int, seed: int, r: int, iterations: int, trace=None):
    """one restart -> (best cost, best step, assignment at that step).  trace(t, pool, cost) sees every state."""
    n = len(w)
    W = np.asarray(w, np.int64)
    perm = list(range(n))
    for k in range(n - 1, 0, -1):
        j = search_hash(seed, r, 0, k) % (k + 1)
        perm[k], perm[j] = perm[j], perm[k]
    pool = np.empty(n, np.int64)
    pool[perm] = np.arange(n) % P
    D = W @ np.eye(P, dtype=np.int64)[pool]                          # D[a][p] = sum of w(a, b), b in pool p
    cost = int(D[np.arange(n), pool].sum()) // 2
    size = np.bincount(pool, minlength=P)
    hi, lo = -(-n // P), n // P
    tabu = np.zeros((n, P), np.int64)
    best, bstep, bpool = cost, 0, pool.copy()
    if trace:
        trace(0, pool, cost)
    ar = np.arange(n)
    for t in range(1, iterations + 1):
        if cost == 0:
            break
        conf = np.nonzero(D[ar, pool] > 0)[0]
        K = len(conf)
        pa = pool[conf]
        keys = []
        delta = (D[conf[:, None], pool[None, :]] - D[conf, pa][:, None] + D[ar[None, :], pa[:, None]]
                 - D[ar, pool][None, :] - 2 * W[conf])
        is_tabu = (tabu[conf[:, None], pool[None, :]] > t) | (tabu[ar[None, :], pa[:, None]] > t)
        ok = (pa[:, None] != pool[None, :]) & (~is_tabu | (cost + delta < best))
        keys.append(((delta + BIAS) << 32 | (conf[:, None] * n + ar[None, :]))[ok])
        if n % P:
            delta = D[conf] - D[conf, pa][:, None]
            ok = ((size[pa] == hi)[:, None] & (size == lo)[None, :]) & (~(tabu[conf] > t) | (cost + delta < best))
            keys.append(((delta + BIAS) << 32 | (n * n + conf[:, None] * P + np.arange(P)[None, :]))[ok])
        keys = np.concatenate(keys)
        if not len(keys):
            break
        key = int(keys.min())
        d, idx = (key >> 32) - BIAS, key & 0xFFFFFFFF
        tenure = 10 + (6 * K) // 10 + search_hash(seed, r, t, 0) % 10
        if idx < n * n:
            a, b = divmod(idx, n)
            qa, qb = int(pool[a]), int(pool[b])
            tabu[a, qa] = tabu[b, qb] = t + tenure
            pool[a], pool[b] = qb, qa
            D[:, qa] += W[:, b] - W[:, a]
            D[:, qb] += W[:, a] - W[:, b]
        else:
            a, q = divmod(idx - n * n, P)
            qa = int(pool[a])
            tabu[a, qa] = t + tenure
            pool[a] = q
            size[qa] -= 1
            size[q] += 1
            D[:, qa] -= W[:, a]
            D[:, q] += W[:, a]
        cost += d
        if trace:
            trace(t, pool, cost)
        if cost < best:
            best, bstep, bpool = cost, t, pool.copy()
    return best, bstep, bpool


def pool_search(w, n_pools, seed, r0, r1, iterations):
    w = np.ascontiguousarray(w, dtype=np.uint8)
    check_args(w, n_pools, r0, r1, iterations)
    out = [restart_search(w, n_pools, int(seed), r, iterations) for r in range(r0, r1)]
    return dict(cost=np.array([o[0] for o in out], np.int64), step=np.array([o[1] for o in out], np.int32),
                assign=np.array([o[2] for o in out], np.uint8).reshape(r1 - r0, len(w)))


class Context(_Context):
    def pool_search(self, w, n_pools, seed, r0, r1, iterations):
        return pool_search(w, n_pools, seed, r0, r1, iterations)
