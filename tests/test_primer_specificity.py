"""primer_specificity end to end against a plain-Python restatement of its semantics (string search on both strands, every
(i, j), no numpy): on the CPU double and on the GPU, in one rank and record-sharded, capped, and its CLI errors.  The
intended groups are also pinned to primer_coverage's amplicons."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.test_primer_coverage import IUPAC, _free_port, find, make_case, rc, read_records, strict_positions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------------------------
def restate_groups(fasta_text, pairs, v, coordinate, lo, hi):
    """(primers [(name, seq)], class [i][j], records, groups {(record, i, j): (products, tot, length, x, lm, rm)})"""
    recs = read_records(fasta_text)
    primers = []
    for name, (f, r) in pairs.items():
        f, r = f.upper(), r.upper()
        fs, _ = strict_positions(coordinate, len(f))
        _, rs = strict_positions(coordinate, len(r))
        primers.append((name + ":F", f, fs))
        primers.append((name + ":R", r, {len(r) - 1 - j for j in rs}))
    intended = set()
    for f, r in pairs.values():
        intended |= {(f.upper(), r.upper()), (r.upper(), f.upper())}
    klass = [["intended" if (a, b) in intended else "self" if a == b else "cross" for _, b, _ in primers]
             for _, a, _ in primers]
    groups = {}
    for t, (_, seq) in enumerate(recs):
        n = len(seq)
        left = [find(seq, p, s, v) for _, p, s in primers]
        right = [[(n - q - len(p), m) for q, m in find(rc(seq), p, s, v)] for _, p, s in primers]
        for i, (_, pi, _) in enumerate(primers):
            for j, (_, pj, _) in enumerate(primers):
                count, best = 0, None
                for x, lm in left[i]:
                    for y, rm in right[j]:
                        length = y + len(pj) - x
                        if y >= x + len(pi) and lo <= length <= hi:
                            count += 1
                            key = (lm + rm, length, x, lm, rm)
                            best = key if best is None or key < best else best
                if count:
                    groups[(t, i, j)] = (count,) + best
    return [(nm, p) for nm, p, _ in primers], klass, recs, groups


def restate(fasta_text, pairs, v, coordinate, lo, hi, max_rows=None):
    """(specificity.tsv, products.tsv) as text"""
    primers, klass, recs, groups = restate_groups(fasta_text, pairs, v, coordinate, lo, hi)
    n = len(recs)
    spec = ["#Left\tRight\tClass\tProducts\tTargets\tPerfect_targets\tTotal\n"]
    unintended, any_t, any_p = 0, set(), set()
    for i in range(len(primers)):
        for j in range(len(primers)):
            mine = [(t, g) for (t, a, b), g in groups.items() if (a, b) == (i, j)]
            if not mine:
                continue
            products = sum(g[0] for _, g in mine)
            perfect = sum(1 for _, g in mine if g[1] == 0)
            spec.append("%s\t%s\t%s\t%d\t%d\t%d\t%d\n" % (primers[i][0], primers[j][0], klass[i][j], products, len(mine),
                                                         perfect, n))
            if klass[i][j] != "intended":
                unintended += products
                any_t |= {t for t, _ in mine}
                any_p |= {t for t, g in mine if g[1] == 0}
    spec.append("UNINTENDED\t-\t-\t%d\t%d\t%d\t%d\n" % (unintended, len(any_t), len(any_p), n))
    prod = ["#Left\tRight\tClass\tTarget\tStart\tEnd\tLength\tLeft_mismatches\tRight_mismatches\tProducts\n"]
    for (t, i, j) in sorted(groups):
        if klass[i][j] == "intended":
            continue
        count, _, length, x, lm, rm = groups[(t, i, j)]
        prod.append("%s\t%s\t%s\t%s\t%d\t%d\t%d\t%d\t%d\t%d\n" % (primers[i][0], primers[j][0], klass[i][j], recs[t][0],
                                                                  x, x + length, length, lm, rm, count))
    if max_rows is not None:
        prod = prod[:1 + max_rows]
    return "".join(spec), "".join(prod)


# ---------------------------------------------------------------------------------------------------------------
# inputs: primer_coverage's case plus self products and a primer listed in two pairs
# ---------------------------------------------------------------------------------------------------------------
def make_spec_case(tmp_path, seed):
    fa, pf, lo, hi = make_case(tmp_path, seed)
    from multiprime_b200.pcr_product import parse_primers
    pairs = parse_primers(pf, "fa")
    rng = np.random.default_rng(seed + 100)
    (f0, r0), (f1, r1) = list(pairs.values())[:2]
    pairs["reuse"] = (f0, r1)                                       # F of pair0 listed in a second pair
    plain = lambda s: "".join(IUPAC[ch][0] for ch in s)           # noqa: E731  (one allowed base per position)
    mid = (lo + hi) // 2
    inv = plain(f1) + "".join(rng.choice(list("ACGT"), mid - 2 * len(f1))) + rc(plain(f1))    # F1 on both strands
    pal = plain(r0) + "".join(rng.choice(list("ACGT"), lo - 2 * len(r0))) + rc(plain(r0))      # exactly lo, i = j
    with open(fa, "a") as fh:
        fh.write(">inverted repeat\n%s\n>self_lo\n%s\n" % (inv, pal))
    pf2 = str(tmp_path / ("primers_spec%d.fa" % seed))
    with open(pf2, "w") as fh:
        fh.write("".join(">%s_F\n%s\n>%s_R\n%s\n" % (n, f, n, r) for n, (f, r) in pairs.items()))
    return fa, pf2, lo, hi


def _run_tool(fa, pf, out, v, lo, hi, backend, comm=None, max_rows=1_000_000):
    from multiprime_b200 import primer_specificity as ps
    from multiprime_b200.pcr_product import parse_primers
    return ps.run(fa, parse_primers(pf, "fa"), out, v, "1,2,-1", (lo, hi), max_rows, comm=comm, _backend=backend)


def _check(tmp_path, fa, pf, lo, hi, v, backend, tag):
    from multiprime_b200.pcr_product import parse_primers
    out = str(tmp_path / tag)
    _run_tool(fa, pf, out, v, lo, hi, backend)
    want_spec, want_prod = restate(open(fa).read(), parse_primers(pf, "fa"), v, "1,2,-1", lo, hi)
    assert open(out + ".specificity.tsv").read() == want_spec
    assert open(out + ".products.tsv").read() == want_prod
    return want_spec, want_prod


def _assert_case_covers(spec, prod, lo, v):
    """the case holds self and cross products, a self product of exactly lo, mismatched sites (v > 0), and the primer
    listed in two pairs forms intended products with the partner of its other pair"""
    rows = [ln.split("\t") for ln in prod.splitlines()[1:]]
    assert {r[2] for r in rows} == {"self", "cross"}
    assert any(r[2] == "self" and r[3] == "self_lo" and int(r[6]) == lo for r in rows)
    assert any(r[2] == "self" and r[3] == "inverted" for r in rows)
    assert any(int(r[7]) + int(r[8]) > 0 for r in rows) == (v > 0)
    srows = [ln.split("\t") for ln in spec.splitlines()[1:-1]]
    reuse_f = [r for r in srows if r[0].startswith("reuse") and r[0].endswith(":F")]
    assert any(r[1].startswith("pair0") and r[1].endswith(":R") and r[2] == "intended" for r in reuse_f)


def _backend(kind):
    if kind == "gpu":
        from multiprime_b200 import _lib
        return _lib
    from tests import fake_pattern_products
    return fake_pattern_products


@pytest.mark.parametrize("stride", [64, None])
@pytest.mark.parametrize("v", [0, 1, 3])
def test_tool_matches_restatement_fake(tmp_path, monkeypatch, stride, v):
    from multiprime_b200 import primer_coverage as pc
    if stride:
        monkeypatch.setattr(pc, "S", stride)
    fa, pf, lo, hi = make_spec_case(tmp_path, seed=v)
    spec, prod = _check(tmp_path, fa, pf, lo, hi, v, _backend("fake"), "fake")
    _assert_case_covers(spec, prod, lo, v)


@pytest.mark.gpu
@pytest.mark.parametrize("stride", [64, None])
@pytest.mark.parametrize("v", [0, 1, 3])
def test_tool_matches_restatement_gpu(tmp_path, monkeypatch, stride, v):
    from multiprime_b200 import primer_coverage as pc
    if stride:
        monkeypatch.setattr(pc, "S", stride)
    fa, pf, lo, hi = make_spec_case(tmp_path, seed=v + 10)
    _check(tmp_path, fa, pf, lo, hi, v, _backend("gpu"), "gpu")


def _intended_matches_coverage(tmp_path, backend, v):
    """the intended groups of pair q, (F_q, R_q) as + and (R_q, F_q) as -, best of both, are primer_coverage's amplicons"""
    from multiprime_b200 import primer_coverage as pc
    from multiprime_b200 import primer_specificity as ps
    from multiprime_b200.pcr_product import parse_primers
    fa, pf, lo, hi = make_spec_case(tmp_path, seed=20 + v)
    pairs = parse_primers(pf, "fa")
    best = pc.run(fa, pairs, str(tmp_path / "cov"), v, "1,2,-1", (lo, hi), _backend=backend)
    targets = pc.read_targets(fa)
    panel = pc.Panel(pairs, "1,2,-1")
    n = 2 * len(panel.names)
    res = ps.find_groups(targets, panel, v, lo, hi, np.ones((n, n), np.uint8), 1 << 30, backend=backend)
    assert res["n_listed"] == len(res["rows"]) == res["stats"][3]
    for q, b in enumerate(best):
        cand = {}
        for rec, i, j, s, ln, lm, rm, _ in res["rows"].tolist():
            if (i, j) in ((2 * q, 2 * q + 1), (2 * q + 1, 2 * q)):
                strand = 0 if i == 2 * q else 1
                fm, rmm = (lm, rm) if strand == 0 else (rm, lm)
                key = (lm + rm, ln, strand, s, fm, rmm)
                cand[rec] = min(cand.get(rec, key), key)
        got = sorted((rec,) + k for rec, k in cand.items())
        want = [(rec, fm + rm, ln, st, s, fm, rm) for rec, st, s, ln, fm, rm in
                zip(*(b[k].tolist() for k in ("rec", "strand", "start", "length", "fmis", "rmis")))]
        assert got == want


@pytest.mark.parametrize("v", [1, 3])
def test_intended_groups_are_coverage_amplicons_fake(tmp_path, v):
    from tests import fake_pattern_products
    _intended_matches_coverage(tmp_path, fake_pattern_products, v)


@pytest.mark.gpu
@pytest.mark.parametrize("v", [1, 3])
def test_intended_groups_are_coverage_amplicons_gpu(tmp_path, v):
    from multiprime_b200 import _lib
    _intended_matches_coverage(tmp_path, _lib, v)


def _max_rows(tmp_path, capsys, backend):
    fa, pf, lo, hi = make_spec_case(tmp_path, seed=4)
    _run_tool(fa, pf, str(tmp_path / "full"), 2, lo, hi, backend)
    full = open(str(tmp_path / "full.products.tsv")).read().splitlines(True)
    assert len(full) > 6
    capsys.readouterr()
    _run_tool(fa, pf, str(tmp_path / "cut"), 2, lo, hi, backend, max_rows=5)
    err = capsys.readouterr().err
    assert "lists 5 of %d rows" % (len(full) - 1) in err
    assert open(str(tmp_path / "cut.products.tsv")).read() == "".join(full[:6])
    assert open(str(tmp_path / "cut.specificity.tsv")).read() == open(str(tmp_path / "full.specificity.tsv")).read()


def test_max_rows_cuts_the_listing_fake(tmp_path, capsys):
    _max_rows(tmp_path, capsys, _backend("fake"))


@pytest.mark.gpu
def test_max_rows_cuts_the_listing_gpu(tmp_path, capsys):
    _max_rows(tmp_path, capsys, _backend("gpu"))


def _sharded(tmp_path, monkeypatch, world, kind):
    """thread shards write the files of one process; world 3 on a case whose first record holds most of the stream
    leaves a rank without a record"""
    from multiprime_b200 import primer_coverage as pc
    from tests.loopback_comm import run_shards
    monkeypatch.setattr(pc, "S", 64)
    fa, pf, lo, hi = make_spec_case(tmp_path, seed=5)
    if world == 3:
        text = open(fa).read()
        recs = read_records(text)
        big = "".join(s for _, s in recs) * 3
        with open(fa, "w") as fh:
            fh.write(">big\n%s\n%s" % (big, text))
        from multiprime_b200 import primer_specificity as ps
        t = pc.read_targets(fa)
        bounds = ps.shard_records(t, 32, 3)
        assert (np.diff(bounds) == 0).any()
    backend = _backend(kind)
    _run_tool(fa, pf, str(tmp_path / "one"), 2, lo, hi, backend)
    run_shards(world, lambda rank, comm: _run_tool(fa, pf, str(tmp_path / "sharded"), 2, lo, hi, backend, comm,
                                                   max_rows=7))
    assert open(str(tmp_path / "one.specificity.tsv")).read() == open(str(tmp_path / "sharded.specificity.tsv")).read()
    one = open(str(tmp_path / "one.products.tsv")).read().splitlines(True)
    assert open(str(tmp_path / "sharded.products.tsv")).read() == "".join(one[:8])


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_threads_write_the_same_files_fake(tmp_path, monkeypatch, world):
    _sharded(tmp_path, monkeypatch, world, "fake")


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_threads_write_the_same_files_gpu(tmp_path, monkeypatch, world):
    _sharded(tmp_path, monkeypatch, world, "gpu")


# ---------------------------------------------------------------------------------------------------------------
# CLI
# ---------------------------------------------------------------------------------------------------------------
def _cli(args, env=None):
    return subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "primer_specificity.py")] + args,
                          capture_output=True, text=True, timeout=300, env=env)


def _cli_error(tmp_path, args, msg):
    fa = tmp_path / "t.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTACGT\n")
    base = {"-r": str(fa), "-i": "ACGTACGTACGTACGTAC,ACGTACGTACGTACGTAC", "-f": "seq", "-o": str(tmp_path / "o")}
    for k, val in zip(args[::2], args[1::2]):
        if val is None:
            del base[k]
        else:
            base[k] = val
    res = _cli([x for kv in base.items() for x in kv])
    assert res.returncode == 1, res.stderr
    assert msg in res.stderr
    assert not os.path.exists(str(tmp_path / "o") + ".specificity.tsv")
    assert not os.path.exists(str(tmp_path / "o") + ".products.tsv")


@pytest.mark.parametrize("args,msg", [
    (["--max-rows", "-1"], "--max-rows must be >= 0"),
    (["-v", "16"], "-v must be in 0..15"),
    (["-s", "500,100"], "0 < lo <= hi"),
    (["-r", None], "Input (targets) file must be specified"),
])
def test_cli_errors(tmp_path, args, msg):
    _cli_error(tmp_path, args, msg)


def test_packing_limit_is_refused_fake(tmp_path):
    from multiprime_b200 import primer_specificity as ps
    from tests import fake_pattern_products
    fa = tmp_path / "t.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTACGT\n")
    with pytest.raises(SystemExit, match="lo <= hi <= 8388607"):
        ps.run(str(fa), {"p": ("ACGTACGTACGTACGTAC", "ACGTACGTACGTACGTAC")}, str(tmp_path / "o"), 1, "1,2,-1",
               (50, 1 << 23), _backend=fake_pattern_products)
    assert not os.path.exists(str(tmp_path / "o") + ".specificity.tsv")


@pytest.mark.gpu
def test_cli_packing_limit_is_refused_gpu(tmp_path):
    _cli_error(tmp_path, ["-s", "50,%d" % (1 << 23)], "lo <= hi <= 8388607")


# ---------------------------------------------------------------------------------------------------------------
# torchrun
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_cli_under_torchrun(tmp_path, backend):
    """two ranks under torchrun write the files of one process: gloo with both ranks on cuda:0, NCCL on two GPUs"""
    import torch
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    fa, pf, lo, hi = make_spec_case(tmp_path, seed=7)
    common = ["-r", fa, "-i", pf, "-f", "fa", "-v", "2", "-s", "%d,%d" % (lo, hi), "--max-rows", "20"]
    one = _cli(common + ["-o", str(tmp_path / "one")])
    assert one.returncode == 0, one.stderr[-3000:]
    env = dict(os.environ, MPB_DIST_BACKEND=backend)
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
                          os.path.join(ROOT, "scripts", "primer_specificity.py")] + common + ["-o", str(tmp_path / "two")],
                         capture_output=True, text=True, env=env, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    assert res.stdout.count("Total times") == 1
    for ext in (".specificity.tsv", ".products.tsv"):
        assert open(str(tmp_path / "one") + ext).read() == open(str(tmp_path / "two") + ext).read()
