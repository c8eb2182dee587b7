"""Split a multiplex primer set into P balanced pools (tubes) with the fewest cross products and primer dimers inside the
pools.  primer_specificity reports what the pairs of a set amplify together and finDimer which primers form dimers;
this tool assigns the pairs to tubes so that conflicting pairs do not share one (tiled amplicon schemes: two
alternating pools).

Semantics
  Primers   Primers, indices (2q = F_q, 2q + 1 = R_q), classes and products are primer_specificity's (Primers,
            find_groups, run with nothing listed).
  Conflicts The weight w(a, b) of pairs a != b counts the conflicting primer combinations between them:
              product  each ordered (i, j), one primer of a and the other of b, of class cross with a product on at
                       least one record (comb[i, j, 1] > 0);
              dimer    each unordered {i, j}, one primer of a and one of b, with different sequences, that finDimer's
                       rule reports (the dimer grid over the set's distinct sequences: ends of 5..18, both initiation
                       terms, loss_table(-t)).
            So 0 <= w <= 12.  Combinations inside one pair, self-class products and dimers of a sequence with itself
            cannot be removed by pooling: they do not count, but <out>.conflicts.tsv lists them.
  Objective Every pair gets a pool, every pool holds floor(n/P) or ceil(n/P) pairs; minimise the cost, the sum of
            w(a, b) over the pairs a < b that share a pool.  Limits: 1 <= P <= 32, P <= n, n <= 512 pairs.
  Search    R restarts r = 0 .. R-1 of a tabu search of at most I steps each (mpb_pool_search, one CTA per restart):
            hash(seed, r, t, k) = mix(mix(seed) ^ (r << 40 | t << 20 | k)) in 64-bit arithmetic, where mix is
            splitmix64's finaliser z ^= z >> 30; z *= 0xbf58476d1ce4e5b9; z ^= z >> 27; z *= 0x94d049bb133111eb;
            z ^= z >> 31 (r < 2^24, t < 2^20, k < 2^20).
            1. Start: the Fisher-Yates shuffle perm = [0 .. n-1], for k = n-1 down to 1 swap perm[k] and
               perm[hash(seed, r, 0, k) mod (k + 1)]; pair perm[k] goes to pool k mod P.
            2. D[a][p] = sum of w(a, b) over the b in pool p; pair a is conflicting when D[a][pool(a)] > 0.
            3. Step t = 1, 2, ..., I, while the cost is > 0.  With K conflicting pairs, the candidates are
                 swap (a, b)  a conflicting, b in another pool; delta = D[a][pb] - D[a][pa] + D[b][pa] - D[b][pb]
                              - 2 w(a, b); index a*n + b;
                 move (a, q)  only when P does not divide n: a conflicting in a pool of ceil(n/P) pairs, q a pool of
                              floor(n/P); delta = D[a][q] - D[a][pa]; index n*n + a*P + q.
               A candidate is tabu when it puts a pair into a pool p while t < tabu[pair][p]; a tabu candidate is
               still admissible when cost + delta < best (the restart's best cost so far).  The admissible candidate
               with the smallest (delta, index) is applied; none ends the restart.  Every pair that leaves a pool p
               gets tabu[pair][p] = t + tenure, tenure = 10 + floor(6K / 10) + hash(seed, r, t, 0) mod 10.
            4. The restart keeps its best cost, the first step that reached it (0: the start) and the assignment then.
            The answer is the restart with the lowest (cost, r); its pools are renumbered 1 .. P by first appearance in
            pair order.  It depends on the inputs and the flags only (not on the GPU, the ranks or the block order).

Under torchrun the specificity search is record-sharded as in primer_specificity, the dimer bands are dealt as in
finDimer, and each rank takes a contiguous block of restarts; rank 0 gathers the (cost, restart, assignment) records
and writes.

Outputs
  <out>.pools.tsv      one row per pair in input order: pool, primers and Conflicts, the pair's share of the cost (sum of
                       w(a, b) over the b in its pool); then a TOTAL row with the cost.
  <out>.conflicts.tsv  one row per conflict between two primers in one pool, by pool: the products (combinations (i, j)
                       with a product that are not intended) in (i, j) order, then the dimers (i <= j) in (i, j) order.
                       Counted is yes when the row counts toward the cost; Targets and Products come from
                       primer_specificity's summary (- for dimers)."""
from __future__ import annotations

import sys
import time
from optparse import SUPPRESS_HELP, OptionParser

import numpy as np

from . import _lib
from . import primer_coverage as pc
from . import primer_specificity as ps
from .findimer import grid_hits
from .iupac import sets_of
from .pcr_product import parse_primers

MAX_PAIRS = 512
MAX_POOLS = 32
MAX_RESTARTS = 1 << 24
MAX_ITERATIONS = (1 << 20) - 1
RESTARTS = 256
ITERATIONS = 2000
SEED = 1
POOLS_HEADER = "#Pair\tPool\tPrimer_F\tPrimer_R\tConflicts\n"
CONFLICTS_HEADER = "#Pool\tLeft\tRight\tKind\tClass\tCounted\tTargets\tProducts\n"
M64 = 0xFFFFFFFFFFFFFFFF


def mix(z: int) -> int:
    """splitmix64's finaliser"""
    z = ((z ^ (z >> 30)) * 0xbf58476d1ce4e5b9) & M64
    z = ((z ^ (z >> 27)) * 0x94d049bb133111eb) & M64
    return z ^ (z >> 31)


def search_hash(seed: int, restart: int, step: int, slot: int) -> int:
    """the counter-based hash of the search (csrc/mpb_pools.cu pool_hash)"""
    return mix(mix(seed & M64) ^ ((restart << 40) | (step << 20) | slot))


def conflict_matrices(primers: ps.Primers, comb, dimer_seq_pairs):
    """(product[i, j], dimer[i, j]) over the primers: combinations with a product that are not intended, and primer
    combinations whose sequences form a dimer (symmetric; the same sequence included)"""
    n = len(primers.seqs)
    product = (comb[:, :, 1] > 0) & (primers.klass != 0)
    index = {}
    for i, s in enumerate(primers.seqs):
        index.setdefault(s, []).append(i)
    dimer = np.zeros((n, n), bool)
    for sa, sb in dimer_seq_pairs:
        for i in index.get(sa, ()):
            for j in index.get(sb, ()):
                dimer[i, j] = dimer[j, i] = True
    return product, dimer


def counted(primers: ps.Primers, product, dimer):
    """(product, dimer) restricted to the combinations that count: primers of different pairs, class cross / different
    sequences"""
    n = len(primers.seqs)
    pair = np.arange(n) // 2
    other = pair[:, None] != pair[None, :]
    seqs = np.array(primers.seqs, dtype=object)
    return product & other & (primers.klass == 2), dimer & other & (seqs[:, None] != seqs[None, :])


def weights(primers: ps.Primers, product, dimer) -> np.ndarray:
    """w[a, b] over the pairs (uint8, symmetric, zero diagonal)"""
    cp, cd = counted(primers, product, dimer)
    n = len(primers.seqs) // 2
    wp = cp.reshape(n, 2, n, 2).sum(axis=(1, 3))
    wd = np.triu(cd).reshape(n, 2, n, 2).sum(axis=(1, 3))       # each unordered {i, j} once
    w = wp + wp.T + wd + wd.T
    np.fill_diagonal(w, 0)
    return w.astype(np.uint8)


def renumber(assign) -> np.ndarray:
    """pools 0 .. P-1 renumbered by first appearance in pair order"""
    first = {}
    for p in assign.tolist():
        first.setdefault(p, len(first))
    return np.array([first[p] for p in assign.tolist()], np.int64)


def pick(cost, restart, assign):
    """the record with the lowest (cost, restart) -> (cost, restart, renumbered assignment)"""
    k = int(np.lexsort((restart, cost))[0])
    return int(cost[k]), int(restart[k]), renumber(assign[k])


def check_pools(n_pairs: int, pools: int, restarts: int, iterations: int):
    if not 1 <= pools <= MAX_POOLS:
        raise SystemExit("Error: -p must be in 1..%d (got %d)" % (MAX_POOLS, pools))
    if n_pairs > MAX_PAIRS:
        raise SystemExit("Error: %d primer pairs: at most %d pairs can be pooled" % (n_pairs, MAX_PAIRS))
    if pools > n_pairs:
        raise SystemExit("Error: -p %d is more pools than the %d primer pairs" % (pools, n_pairs))
    if not 1 <= restarts <= MAX_RESTARTS:
        raise SystemExit("Error: --restarts must be in 1..%d (got %d)" % (MAX_RESTARTS, restarts))
    if not 0 <= iterations <= MAX_ITERATIONS:
        raise SystemExit("Error: --iterations must be in 0..%d (got %d)" % (MAX_ITERATIONS, iterations))


def search(ctx, w, pools: int, seed: int, restarts: int, iterations: int, comm=None):
    """every rank runs a contiguous block of the restarts; -> (cost, restart, assignment) of the answer on rank 0, None
    on the other ranks"""
    rank, world = (comm.rank, comm.world) if comm is not None else (0, 1)
    n = len(w)
    r0, r1 = restarts * rank // world, restarts * (rank + 1) // world
    res = ctx.pool_search(w, pools, seed, r0, r1, iterations)
    recs = np.concatenate([res["cost"][:, None], np.arange(r0, r1, dtype=np.int64)[:, None],
                           res["assign"].astype(np.int64)], axis=1).reshape(-1)
    if comm is not None and world > 1:
        recs, _ = comm.allgather_concat(recs)
        if rank != 0:
            return None
    recs = recs.reshape(-1, n + 2)
    return pick(recs[:, 0], recs[:, 1], recs[:, 2:])


def write_outputs(out: str, panel: pc.Panel, primers: ps.Primers, comb, product, dimer, w, pool):
    n = len(panel.names)
    same = pool[:, None] == pool[None, :]
    share = (w.astype(np.int64) * same).sum(axis=1)
    with open(out + ".pools.tsv", "w") as fo:
        fo.write(POOLS_HEADER)
        for a, name in enumerate(panel.names):
            fo.write("%s\t%d\t%s\t%s\t%d\n" % (name, pool[a] + 1, panel.primers[a][0], panel.primers[a][1], share[a]))
        fo.write("TOTAL\t-\t-\t-\t%d\n" % (int(share.sum()) // 2))
    cp, cd = counted(primers, product, dimer)
    ppool = np.repeat(pool, 2)
    names, kinds = primers.names, ps.CLASSES
    with open(out + ".conflicts.tsv", "w") as fo:
        fo.write(CONFLICTS_HEADER)
        for p in range(int(pool.max()) + 1 if n else 0):
            mine = ppool == p
            inside = mine[:, None] & mine[None, :]
            for i, j in zip(*np.nonzero(product & inside)):
                fo.write("%d\t%s\t%s\tproduct\t%s\t%s\t%d\t%d\n" % (p + 1, names[i], names[j], kinds[primers.klass[i, j]],
                                                                   "yes" if cp[i, j] else "no", comb[i, j, 1],
                                                                   comb[i, j, 0]))
            for i, j in zip(*np.nonzero(np.triu(dimer & inside))):
                fo.write("%d\t%s\t%s\tdimer\t%s\t%s\t-\t-\n" % (p + 1, names[i], names[j], kinds[primers.klass[i, j]],
                                                               "yes" if cd[i, j] else "no"))


def run(ref: str, pairs: dict, out: str, v: int = 1, coordinate: str = "1,2,-1", size=(50, 2000), pools: int = 2,
        threshold: float = 3.96, restarts: int = RESTARTS, iterations: int = ITERATIONS, seed: int = SEED, device=0,
        comm=None, _backend=None, _times=None):
    """-> dict(cost, restart, pool int64[n] (0-based), w) on rank 0, None on the other ranks"""
    backend = _backend or _lib
    lo, hi = size
    panel = pc.Panel(pairs, coordinate)
    if not panel.names:
        raise SystemExit("Error: no primer pair in the primer file")
    pc.check_limits(panel, v, lo, hi)
    check_pools(len(panel.names), pools, restarts, iterations)
    times = _times if _times is not None else {}
    t0 = time.perf_counter()
    targets = pc.read_targets(ref)
    primers = ps.Primers(panel)
    n_primer = len(primers.seqs)
    try:
        t1 = time.perf_counter()
        res = ps.find_groups(targets, panel, v, lo, hi, np.zeros((n_primer, n_primer), np.uint8), 0, device, comm,
                             backend)
        t2 = time.perf_counter()
        ctx = backend.Context.shared(device)
        distinct = sorted(set(primers.seqs), key=primers.seqs.index)
        hits, _, _ = grid_hits(ctx, backend, [sets_of(s) for s in distinct], threshold, comm)
        t3 = time.perf_counter()
        comb = res["comb"] if res is not None else np.zeros((n_primer, n_primer, 3), np.int64)
        if comm is not None and comm.world > 1:          # the summary lives on rank 0; every rank needs w
            comb = comm.allreduce_sum(comb.reshape(-1)).reshape(n_primer, n_primer, 3)
        product, dimer = conflict_matrices(primers, comb, [(distinct[i], distinct[j]) for i, j, _, _ in hits])
        w = weights(primers, product, dimer)
        found = search(ctx, w, pools, seed, restarts, iterations, comm)
        t4 = time.perf_counter()
    except _lib.MpbError as exc:
        raise SystemExit("Error: %s" % exc)
    times.update(read=t1 - t0, specificity=t2 - t1, dimer=t3 - t2, search=t4 - t3)
    if found is None:
        return None
    cost, restart, pool = found
    write_outputs(out, panel, primers, comb, product, dimer, w, pool)
    return dict(cost=cost, restart=restart, pool=pool, w=w)


def argsParse(argv=None):
    parser = OptionParser('Usage: %prog -r [targets.fa] -i [primers] -f [format] -o [out_prefix] -p [pools]')
    ps.add_options(parser, "primer_pools", "<out>.pools.tsv and <out>.conflicts.tsv")
    parser.add_option('-p', '--pools', dest='pools', default=2, type="int", help='Number of pools (tubes). Default: 2.')
    parser.add_option('-t', '--threshold', dest='threshold', default=3.96, type="float",
                      help='Threshold of the dimer loss function (finDimer -t). Default: 3.96.')
    parser.add_option('--restarts', dest='restarts', default=RESTARTS, type="int",
                      help='Independent restarts of the pool search. Default: %d.' % RESTARTS)
    parser.add_option('--iterations', dest='iterations', default=ITERATIONS, type="int",
                      help='Steps of each restart at most. Default: %d.' % ITERATIONS)
    parser.add_option('--seed', dest='seed', default=SEED, type="int", help='Seed of the search. Default: %d.' % SEED)
    parser.add_option('--device', dest='device', default=0, type="int", help=SUPPRESS_HELP)
    args = sys.argv[1:] if argv is None else argv
    (options, rest) = parser.parse_args(args)
    return ps.check_options(parser, options)


def main(argv=None, _backend=None):
    from .findimer import shard_setup
    e1 = time.time()
    options = argsParse(argv)
    extra, rank = shard_setup(options.device)
    res = run(options.ref, parse_primers(options.input, options.format), options.out, options.variation,
              options.coordinate, options.size, options.pools, options.threshold, options.restarts, options.iterations,
              options.seed, _backend=_backend, **extra)
    if "comm" in extra:
        import torch.distributed as dist
        dist.destroy_process_group()
    e2 = time.time()
    if rank == 0:
        print("INFO {} Pools: {} Cost: {} Restarts: {} Iterations: {} Total times: {}".format(
            time.strftime("%Y-%m-%d %H:%M:%S", time.localtime(time.time())), options.pools, res["cost"],
            options.restarts, options.iterations, round(float(e2 - e1), 2)))


if __name__ == "__main__":
    main()
