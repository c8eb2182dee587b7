"""primer_pools end to end against a plain-Python restatement: w rebuilt from primer_specificity's specificity.tsv and
finDimer's rows, the chosen restart formatted by hand; on the CPU double and on the GPU, in one rank, thread-sharded and
under torchrun.  Also: each pool's own specificity run lists exactly the pool's product rows, a tiled panel splits into
two alternating pools, and the CLI's refusals."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.test_primer_coverage import _free_port, rc
from tests.test_primer_specificity import make_spec_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARGS = dict(pools=2, threshold=3.96, restarts=6, iterations=200, seed=3)


def _backend(kind):
    if kind == "gpu":
        from multiprime_b200 import _lib
        return _lib
    from tests import fake_pool_search
    return fake_pool_search


# ---------------------------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------------------------
def restate(tmp_path, fa, pairs, v, lo, hi, backend, pools, threshold, restarts, iterations, seed):
    """(pools.tsv, conflicts.tsv) as text"""
    from multiprime_b200 import primer_specificity as ps
    from multiprime_b200.findimer import Dimer
    from tests import fake_pool_search as fps
    spec_out = str(tmp_path / "restate_spec")
    ps.run(fa, pairs, spec_out, v, "1,2,-1", (lo, hi), 0, _backend=backend)
    spec = {}
    for line in open(spec_out + ".specificity.tsv").read().splitlines()[1:-1]:
        left, right, klass, products, targets = line.split("\t")[:5]
        spec[(left, right)] = (klass, products, targets)
    names, seqs = [], []
    for q, (f, r) in pairs.items():
        names += [q + ":F", q + ":R"]
        seqs += [f.strip().upper(), r.strip().upper()]
    distinct = []
    for s in seqs:
        if s not in distinct:
            distinct.append(s)
    dfa = tmp_path / "restate_distinct.fa"
    dfa.write_text("".join(">s%d\n%s\n" % (k, s) for k, s in enumerate(distinct)))
    rows = Dimer(str(dfa), str(tmp_path / "restate_dimer"), threshold, ctx=backend.Context(0), _backend=backend).find()
    dimers = {frozenset((r[1], r[8])) for r in rows}
    n = len(names) // 2

    def is_dimer(i, j):
        return frozenset((seqs[i], seqs[j])) in dimers

    def counted_product(i, j):
        return i // 2 != j // 2 and spec.get((names[i], names[j]), ("",))[0] == "cross"

    def counted_dimer(i, j):
        return i // 2 != j // 2 and seqs[i] != seqs[j] and is_dimer(i, j)

    w = np.zeros((n, n), np.uint8)
    for a in range(n):
        for b in range(n):
            if a != b:
                for i in (2 * a, 2 * a + 1):
                    for j in (2 * b, 2 * b + 1):
                        w[a, b] += counted_product(i, j) + counted_product(j, i) + counted_dimer(i, j)
    res = fps.pool_search(w, pools, seed, 0, restarts, iterations)
    best = min(range(restarts), key=lambda r: (int(res["cost"][r]), r))
    first = {}
    for p in res["assign"][best].tolist():
        first.setdefault(p, len(first))
    pool = [first[p] for p in res["assign"][best].tolist()]
    out = ["#Pair\tPool\tPrimer_F\tPrimer_R\tConflicts\n"]
    total = 0
    for a, q in enumerate(pairs):
        share = sum(int(w[a, b]) for b in range(n) if pool[b] == pool[a])
        total += share
        out.append("%s\t%d\t%s\t%s\t%d\n" % (q, pool[a] + 1, seqs[2 * a], seqs[2 * a + 1], share))
    out.append("TOTAL\t-\t-\t-\t%d\n" % (total // 2))
    conf = ["#Pool\tLeft\tRight\tKind\tClass\tCounted\tTargets\tProducts\n"]
    klass = {}
    for i in range(2 * n):
        for j in range(2 * n):
            intended = any((seqs[i], seqs[j]) in ((f.upper(), r.upper()), (r.upper(), f.upper()))
                           for f, r in pairs.values())
            klass[i, j] = "intended" if intended else "self" if seqs[i] == seqs[j] else "cross"
    for p in range(max(pool) + 1):
        mine = [i for i in range(2 * n) if pool[i // 2] == p]
        for i in mine:
            for j in mine:
                if (names[i], names[j]) in spec and spec[(names[i], names[j])][0] != "intended":
                    k, products, targets = spec[(names[i], names[j])]
                    conf.append("%d\t%s\t%s\tproduct\t%s\t%s\t%s\t%s\n" % (p + 1, names[i], names[j], k,
                                                                           "yes" if counted_product(i, j) else "no",
                                                                           targets, products))
        for i in mine:
            for j in mine:
                if i <= j and is_dimer(i, j):
                    conf.append("%d\t%s\t%s\tdimer\t%s\t%s\t-\t-\n" % (p + 1, names[i], names[j], klass[i, j],
                                                                       "yes" if counted_dimer(i, j) else "no"))
    return "".join(out), "".join(conf)


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def make_pool_case(tmp_path, seed):
    """primer_specificity's case (a primer listed in two pairs, self products) plus a pair whose R is the reverse
    complement of its F (an intra-pair dimer) and a pair that forms a dimer with pair0's F"""
    from multiprime_b200.pcr_product import parse_primers
    fa, pf, lo, hi = make_spec_case(tmp_path, seed)
    pairs = parse_primers(pf, "fa")
    rng = np.random.default_rng(seed + 300)
    rand = lambda k: "".join(rng.choice(list("ACGT"), k))       # noqa: E731
    hair = rand(22)
    pairs["hairpin"] = (hair, rc(hair))
    f0 = list(pairs.values())[0][0]
    pairs["partner"] = (rand(12) + rc("".join(c if c in "ACGT" else "A" for c in f0[-10:])), rand(21))
    pf2 = str(tmp_path / ("primers_pool%d.fa" % seed))
    with open(pf2, "w") as fh:
        fh.write("".join(">%s_F\n%s\n>%s_R\n%s\n" % (n, f, n, r) for n, (f, r) in pairs.items()))
    return fa, pf2, lo, hi


def _run_tool(fa, pf, out, lo, hi, backend, comm=None, v=1, **kw):
    from multiprime_b200 import primer_pools as pp
    from multiprime_b200.pcr_product import parse_primers
    args = dict(ARGS, **kw)
    return pp.run(fa, parse_primers(pf, "fa"), out, v, "1,2,-1", (lo, hi), args["pools"], args["threshold"],
                  args["restarts"], args["iterations"], args["seed"], comm=comm, _backend=backend)


def _check(tmp_path, kind, seed, v=1, **kw):
    from multiprime_b200.pcr_product import parse_primers
    backend = _backend(kind)
    fa, pf, lo, hi = make_pool_case(tmp_path, seed)
    out = str(tmp_path / kind)
    _run_tool(fa, pf, out, lo, hi, backend, v=v, **kw)
    args = dict(ARGS, **kw)
    want_pools, want_conf = restate(tmp_path, fa, parse_primers(pf, "fa"), v, lo, hi, backend, args["pools"],
                                    args["threshold"], args["restarts"], args["iterations"], args["seed"])
    got_pools, got_conf = open(out + ".pools.tsv").read(), open(out + ".conflicts.tsv").read()
    assert got_pools == want_pools
    assert got_conf == want_conf
    return got_pools, got_conf


def _assert_case_covers(conf):
    rows = [ln.split("\t") for ln in conf.splitlines()[1:]]
    assert any(r[3] == "product" and r[4] == "self" and r[5] == "no" for r in rows)
    assert any(r[3] == "dimer" and r[1].startswith("hairpin") and r[2].startswith("hairpin") and r[5] == "no"
               for r in rows)
    assert all(r[5] == "no" for r in rows if r[1].split(":")[0] == r[2].split(":")[0])


@pytest.mark.parametrize("pools", [1, 2, 3])
def test_tool_matches_restatement_fake(tmp_path, pools):
    _, conf = _check(tmp_path, "fake", 1, pools=pools)
    if pools == 1:
        _assert_case_covers(conf)


@pytest.mark.gpu
@pytest.mark.parametrize("pools", [1, 2, 3])
def test_tool_matches_restatement_gpu(tmp_path, pools):
    _, conf = _check(tmp_path, "gpu", 1, pools=pools)
    if pools == 1:
        _assert_case_covers(conf)


def _pools_list_their_products(tmp_path, kind):
    """primer_specificity on one pool's pairs lists exactly that pool's product rows"""
    from multiprime_b200 import primer_specificity as ps
    from multiprime_b200.pcr_product import parse_primers
    backend = _backend(kind)
    fa, pf, lo, hi = make_pool_case(tmp_path, 2)
    pairs = parse_primers(pf, "fa")
    _run_tool(fa, pf, str(tmp_path / "all"), lo, hi, backend, pools=3)
    pool_of = {ln.split("\t")[0]: ln.split("\t")[1] for ln in open(str(tmp_path / "all.pools.tsv")).read().splitlines()[1:-1]}
    conf = [ln.split("\t") for ln in open(str(tmp_path / "all.conflicts.tsv")).read().splitlines()[1:]]
    for p in sorted(set(pool_of.values())):
        mine = {q: fr for q, fr in pairs.items() if pool_of[q] == p}
        ps.run(fa, mine, str(tmp_path / ("p" + p)), 1, "1,2,-1", (lo, hi), 0, _backend=backend)
        spec = [ln.split("\t") for ln in open(str(tmp_path / ("p%s.specificity.tsv" % p))).read().splitlines()[1:-1]]
        want = [(r[0], r[1], r[2], r[4], r[3]) for r in spec if r[2] != "intended"]
        got = [(r[1], r[2], r[4], r[6], r[7]) for r in conf if r[0] == p and r[3] == "product"]
        assert got == want


def test_pools_list_their_products_fake(tmp_path):
    _pools_list_their_products(tmp_path, "fake")


@pytest.mark.gpu
def test_pools_list_their_products_gpu(tmp_path):
    _pools_list_their_products(tmp_path, "gpu")


def make_tiled(tmp_path, n_pairs=8, step=300, span=400):
    """pairs tiled along one genome, neighbours overlapping: only neighbours form products within 50..500"""
    rng = np.random.default_rng(11)
    genome = "".join(rng.choice(list("ACGT"), step * n_pairs + span + 200))
    pairs = {}
    for q in range(n_pairs):
        a = 100 + q * step
        pairs["tile%d" % q] = (genome[a:a + 20], rc(genome[a + span - 20:a + span]))
    fa = tmp_path / "genome.fa"
    fa.write_text(">genome\n%s\n" % genome)
    pf = tmp_path / "tiles.fa"
    pf.write_text("".join(">%s_F\n%s\n>%s_R\n%s\n" % (n, f, n, r) for n, (f, r) in pairs.items()))
    return str(fa), str(pf)


def test_tiled_panel_alternates_in_two_pools(tmp_path):
    from multiprime_b200.primer_pools import weights  # noqa: F401
    fa, pf = make_tiled(tmp_path)
    res = _run_tool(fa, pf, str(tmp_path / "tiled"), 50, 500, _backend("fake"), v=0, pools=2)
    w = res["w"]
    n = len(w)
    assert all(w[q, q + 1] > 0 for q in range(n - 1))
    assert not np.triu(w, 2).any()
    assert res["cost"] == 0
    assert res["pool"].tolist() == [q % 2 for q in range(n)]
    rows = open(str(tmp_path / "tiled.pools.tsv")).read().splitlines()
    assert [r.split("\t")[1] for r in rows[1:-1]] == [str(1 + q % 2) for q in range(n)]
    assert rows[-1] == "TOTAL\t-\t-\t-\t0"


def _sharded(tmp_path, world, kind):
    from tests.loopback_comm import run_shards
    backend = _backend(kind)
    fa, pf, lo, hi = make_pool_case(tmp_path, 4)
    _run_tool(fa, pf, str(tmp_path / "one"), lo, hi, backend, pools=3, restarts=7)
    run_shards(world, lambda rank, comm: _run_tool(fa, pf, str(tmp_path / "sharded"), lo, hi, backend, comm, pools=3,
                                                   restarts=7))
    for ext in (".pools.tsv", ".conflicts.tsv"):
        assert open(str(tmp_path / "one") + ext).read() == open(str(tmp_path / "sharded") + ext).read()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_threads_write_the_same_files_fake(tmp_path, world):
    _sharded(tmp_path, world, "fake")


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_threads_write_the_same_files_gpu(tmp_path, world):
    _sharded(tmp_path, world, "gpu")


# ---------------------------------------------------------------------------------------------------------------
# CLI
# ---------------------------------------------------------------------------------------------------------------
def _cli(args, env=None):
    return subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "primer_pools.py")] + args,
                          capture_output=True, text=True, timeout=600, env=env)


@pytest.mark.parametrize("args,msg", [
    (["-p", "3"], "-p 3 is more pools than the 2 primer pairs"),
    (["-p", "33"], "-p must be in 1..32"),
    (["-p", "0"], "-p must be in 1..32"),
    (["--restarts", "0"], "--restarts must be in"),
    (["--iterations", "-1"], "--iterations must be in"),
    (["-f", "bad"], "-f must be xls, fa or seq"),
    (["-s", "500"], "-s takes lo,hi"),
    (["-r", None], "Input (targets) file must be specified"),
])
def test_cli_errors(tmp_path, args, msg):
    fa = tmp_path / "t.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTACGT\n")
    base = {"-r": str(fa), "-i": str(tmp_path / "p.fa"), "-f": "fa", "-o": str(tmp_path / "o")}
    (tmp_path / "p.fa").write_text(">a_F\nACGTACGTACGTACGTAC\n>a_R\nTTGCATTGCATTGCATTG\n"
                                   ">b_F\nGGGTACGTACGTACGTAC\n>b_R\nTTGCATTGCATTGCAGGG\n")
    for k, val in zip(args[::2], args[1::2]):
        if val is None:
            del base[k]
        else:
            base[k] = val
    res = _cli([x for kv in base.items() for x in kv])
    assert res.returncode == 1, res.stderr
    assert msg in res.stderr
    assert not os.path.exists(str(tmp_path / "o") + ".pools.tsv")


def test_cli_bad_flag(tmp_path):
    res = _cli(["--no-such-flag"])
    assert res.returncode == 2 and "no such option" in res.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_cli_under_torchrun(tmp_path, backend):
    """two and three ranks under torchrun write the files of one process (gloo with the ranks on cuda:0, NCCL on two
    GPUs), and a second run writes the same files"""
    import torch
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    fa, pf, lo, hi = make_pool_case(tmp_path, 7)
    common = ["-r", fa, "-i", pf, "-f", "fa", "-v", "2", "-s", "%d,%d" % (lo, hi), "-p", "3", "--restarts", "13"]
    one = _cli(common + ["-o", str(tmp_path / "one")])
    assert one.returncode == 0, one.stderr[-3000:]
    assert "Pools: 3 Cost:" in one.stdout
    again = _cli(common + ["-o", str(tmp_path / "again")])
    assert again.returncode == 0, again.stderr[-3000:]
    env = dict(os.environ, MPB_DIST_BACKEND=backend)
    worlds = [2] if backend == "nccl" else [2, 3]
    for world in worlds:
        tag = "w%d" % world
        res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node",
                              str(world), "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
                              os.path.join(ROOT, "scripts", "primer_pools.py")] + common + ["-o", str(tmp_path / tag)],
                             capture_output=True, text=True, env=env, timeout=600)
        assert res.returncode == 0, res.stderr[-3000:]
        assert res.stdout.count("Total times") == 1
        for ext in (".pools.tsv", ".conflicts.tsv"):
            assert open(str(tmp_path / "one") + ext).read() == open(str(tmp_path / tag) + ext).read()
            assert open(str(tmp_path / "one") + ext).read() == open(str(tmp_path / "again") + ext).read()
