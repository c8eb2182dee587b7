"""primer_select end to end against a plain-Python restatement: A(c) and P(c) from test_primer_coverage's str-slicing
restatement, dimers from oracle/dimer_oracle.py's finDimer rule, the greedy on Python sets and the three files formatted
by hand; on the CPU double and on the GPU, in one rank, thread-sharded and under torchrun.  Also: the selected pairs
re-checked by primer_coverage, the sets format, small pair blocks and the CLI's refusals."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.test_primer_coverage import _free_port, make_case, rc, restate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THRESHOLD = 3.96


def _backend(kind):
    if kind == "gpu":
        from multiprime_b200 import _lib
        return _lib
    from tests import fake_pattern_cover
    return fake_pattern_cover


# ---------------------------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------------------------
def restate_select(fa, cands, keep, v, lo, hi, max_pairs=0, goal=1.0, threshold=THRESHOLD):
    """(selected.tsv, candidates.tsv, selected.fa) as text; cands / keep: {name: (F, R)}"""
    from oracle.dimer_oracle import find_dimers
    rows = [(n, f.strip().upper(), r.strip().upper()) for n, (f, r) in keep.items()]
    rows += [(n, f.strip().upper(), r.strip().upper()) for n, (f, r) in cands.items() if n not in keep]
    row_of = {n: i for i, (n, _, _) in enumerate(rows)}
    amp_text, _ = restate(open(fa).read(), {str(i): (f, r) for i, (_, f, r) in enumerate(rows)}, v, "1,2,-1", lo, hi)
    n_targets = sum(1 for ln in open(fa) if ln.startswith(">"))
    A = [set() for _ in rows]
    P = [set() for _ in rows]
    for ln in amp_text.splitlines()[1:]:
        q, target, _, _, _, _, fm, rm = ln.split("\t")
        A[int(q)].add(target)
        if int(fm) + int(rm) == 0:
            P[int(q)].add(target)
    seqs = []
    for _, f, r in rows:
        for s in (f, r):
            if s not in seqs:
                seqs.append(s)
    dimers = {frozenset((d[1], d[8])) for d in find_dimers({s: ">s%d" % k for k, s in enumerate(seqs)}, threshold)}

    def conflict(a, b):
        return a != b and any(sa != sb and frozenset((sa, sb)) in dimers for sa in rows[a][1:] for sb in rows[b][1:])

    covered, covered_p = set(), set()
    taken, excluded, status = [], {}, {}

    def take(q, step):
        new, newp = A[q] - covered, P[q] - covered_p
        covered.update(A[q])
        covered_p.update(P[q])
        taken.append((q, step, len(new), len(newp), len(covered), len(covered_p)))
        for c in range(len(keep), len(rows)):
            if c not in excluded and all(c != t[0] for t in taken) and conflict(q, c):
                excluded[c] = (step, q)

    for q in range(len(keep)):
        take(q, 0)
    step = 0
    while not (max_pairs and step >= max_pairs) and len(covered) / n_targets < goal:
        best = None
        for c in range(len(keep), len(rows)):
            if c in excluded or any(c == t[0] for t in taken):
                continue
            key = (len(A[c] - covered), len(P[c] - covered_p))
            if key[0] > 0 and (best is None or key > best[0]):
                best = (key, c)
        if best is None:
            break
        step += 1
        take(best[1], step)
    sel = ["#Step\tPair\tPrimer_F\tPrimer_R\tAmplified\tPerfect\tNew\tNew_perfect\tCovered\tCovered_perfect\tTotal\t"
           "Coverage\n"]
    fasta = []
    for q, s, new, newp, cov, covp in taken:
        n, f, r = rows[q]
        sel.append("%d\t%s\t%s\t%s\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%s\n" % (s, n, f, r, len(A[q]), len(P[q]), new, newp, cov,
                                                                          covp, n_targets, round(cov / n_targets, 4)))
        fasta.append(">%s:F\n%s\n>%s:R\n%s\n" % (n, f, n, r))
    cand = ["#Pair\tPrimer_F\tPrimer_R\tAmplified\tPerfect\tStatus\tStep\tBy\n"]
    step_of = {t[0]: t[1] for t in taken}
    for name in cands:
        q = row_of[name]
        if q < len(keep):
            st = ("kept", "0", "-")
        elif q in step_of:
            st = ("selected", str(step_of[q]), "-")
        elif q in excluded:
            st = ("dimer", str(excluded[q][0]), rows[excluded[q][1]][0])
        else:
            st = ("open", "-", "-")
        cand.append("%s\t%s\t%s\t%d\t%d\t%s\t%s\t%s\n" % ((name,) + rows[q][1:] + (len(A[q]), len(P[q])) + st))
    return "".join(sel), "".join(cand), "".join(fasta)


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def make_select_case(tmp_path, seed):
    """(fasta, candidates {name: (F, R)}, lo, hi): primer_coverage's case (targets cut from one root) with a pool cut
    from the same root: its three pairs and a copy of pair1; xmm, X with one mismatch in F, before X (equal gains broken
    by the perfect gain); Z, whose R is the reverse complement of X's F (a dimer between two good pairs); W and a copy of
    it under another name (a tie broken by index); and a pair that amplifies nothing (the zero-gain stop)"""
    from multiprime_b200.pcr_product import parse_primers
    fa, pf, lo, hi = make_case(tmp_path, seed)
    root = "".join(np.random.default_rng(seed).choice(list("ACGT"), 1400))   # make_case's first draw
    cands = dict(parse_primers(pf, "fa"))
    cands["pair1_copy"] = cands["pair1_F_pair1_R"]
    xf, xr = root[300:320], rc(root[800:820])
    swap = {"A": "C", "C": "G", "G": "T", "T": "A"}
    cands["xmm"] = (xf[:10] + swap[xf[10]] + xf[11:], xr)
    cands["X"] = (xf, xr)
    cands["Z"] = (root[100:120], rc(xf))
    cands["W"] = (root[900:920], rc(root[1250:1270]))
    cands["W_copy"] = cands["W"]
    rng = np.random.default_rng(seed + 77)
    cands["nothing"] = ("".join(rng.choice(list("ACGT"), 20)), "".join(rng.choice(list("ACGT"), 20)))
    return fa, cands, lo, hi


def _run(fa, cands, out, lo, hi, backend, v=1, comm=None, keep=None, **kw):
    from multiprime_b200 import primer_select as sel
    return sel.run(fa, cands, out, v, "1,2,-1", (lo, hi), kw.get("max_pairs", 0), kw.get("goal", 1.0), THRESHOLD, keep,
                   comm=comm, _backend=backend, _block=kw.get("block", 0))


def _files(out):
    return tuple(open(out + ext).read() for ext in (".selected.tsv", ".candidates.tsv", ".selected.fa"))


def _check(tmp_path, kind, seed=1, v=1, keep=None, **kw):
    fa, cands, lo, hi = make_select_case(tmp_path, seed)
    keep = {k: cands[k] for k in (keep or [])}
    out = str(tmp_path / kind)
    _run(fa, cands, out, lo, hi, _backend(kind), v, keep=keep, **kw)
    want = restate_select(fa, cands, keep, v, lo, hi, kw.get("max_pairs", 0), kw.get("goal", 1.0))
    got = _files(out)
    assert got == want
    return got


def _assert_case_covers(cand_text):
    rows = {r.split("\t")[0]: r.split("\t") for r in cand_text.splitlines()[1:]}
    assert rows["W"][5] == "selected" and rows["W_copy"][5] == "open" and rows["W"][3:5] == rows["W_copy"][3:5]
    assert rows["X"][5] == "selected" and rows["xmm"][5] == "open"
    assert rows["xmm"][3] == rows["X"][3] and int(rows["xmm"][4]) < int(rows["X"][4])
    assert rows["Z"][5] == "dimer" and rows["Z"][7] == "X" and int(rows["Z"][6]) >= 1
    assert rows["nothing"][3] == "0" and rows["nothing"][5] == "open"


CASES = [dict(v=1), dict(v=3, stride=64), dict(v=0)]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_tool_matches_restatement_fake(tmp_path, monkeypatch, case):
    from multiprime_b200 import primer_coverage as pc
    args = dict(CASES[case])
    if args.pop("stride", None):
        monkeypatch.setattr(pc, "S", 64)
    _, cand, _ = _check(tmp_path, "fake", **args)
    if args["v"] == 1:
        _assert_case_covers(cand)


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(CASES)))
def test_tool_matches_restatement_gpu(tmp_path, monkeypatch, case):
    from multiprime_b200 import primer_coverage as pc
    args = dict(CASES[case])
    if args.pop("stride", None):
        monkeypatch.setattr(pc, "S", 64)
    _, cand, _ = _check(tmp_path, "gpu", **args)
    if args["v"] == 1:
        _assert_case_covers(cand)


FLAGS = [dict(keep=["W", "pair2_F_pair2_R"]), dict(keep=["X"]), dict(max_pairs=1), dict(max_pairs=2, goal=0.5),
         dict(goal=0.2), dict(block=1), dict(block=3, keep=["Z"])]


@pytest.mark.parametrize("flags", range(len(FLAGS)))
def test_flags_match_restatement_fake(tmp_path, flags):
    sel, cand, _ = _check(tmp_path, "fake", **FLAGS[flags])
    if FLAGS[flags].get("keep") == ["X"]:          # Z is excluded by a kept pair at step 0
        assert "\tdimer\t0\tX\n" in cand


@pytest.mark.gpu
@pytest.mark.parametrize("flags", range(len(FLAGS)))
def test_flags_match_restatement_gpu(tmp_path, flags):
    _check(tmp_path, "gpu", **FLAGS[flags])


def test_keep_outside_the_pool_fake(tmp_path):
    """a kept pair that is not a candidate is taken at step 0 and listed in selected.tsv only"""
    fa, cands, lo, hi = make_select_case(tmp_path, 1)
    keep = {"panel_old": cands.pop("W")}
    out = str(tmp_path / "k")
    _run(fa, cands, out, lo, hi, _backend("fake"), keep=keep)
    assert _files(out) == restate_select(fa, cands, keep, 1, lo, hi)
    assert _files(out)[0].splitlines()[1].startswith("0\tpanel_old\t")
    assert "panel_old" not in _files(out)[1]


def _cross_check(tmp_path, kind):
    """Amplified / Perfect of selected.tsv and the last Covered / Covered_perfect equal primer_coverage.run on the
    selected pairs read back from selected.fa"""
    from multiprime_b200 import primer_coverage as pc
    from multiprime_b200.pcr_product import parse_primers
    fa, cands, lo, hi = make_select_case(tmp_path, 2)
    out = str(tmp_path / "sel")
    _run(fa, cands, out, lo, hi, _backend(kind), v=2)
    back = parse_primers(out + ".selected.fa", "fa")
    backend = _backend(kind)
    if kind == "fake":
        from tests import fake_pattern_sites as backend
    pc.run(fa, back, str(tmp_path / "cov"), 2, "1,2,-1", (lo, hi), _backend=backend)
    sel = [r.split("\t") for r in open(out + ".selected.tsv").read().splitlines()[1:]]
    cov = [r.split("\t") for r in open(str(tmp_path / "cov.coverage.tsv")).read().splitlines()[1:]]
    assert len(sel) >= 2
    assert [(s[1] + ":F_" + s[1] + ":R", s[2], s[3], s[4], s[5]) for s in sel] == [tuple(c[:5]) for c in cov[:-1]]
    assert (sel[-1][8], sel[-1][9]) == (cov[-1][3], cov[-1][4])


def test_cross_check_with_primer_coverage_fake(tmp_path):
    _cross_check(tmp_path, "fake")


@pytest.mark.gpu
def test_cross_check_with_primer_coverage_gpu(tmp_path):
    _cross_check(tmp_path, "gpu")


def test_sets_format(tmp_path):
    """get_multiPrime's sets file: pairs named as parse_primers names them in an xls, a repeated name skipped, empty
    fields dropped, an incomplete last group ignored"""
    from multiprime_b200 import primer_select as sel
    fa, cands, lo, hi = make_select_case(tmp_path, 1)
    items = [tuple(fr) for fr in cands.values()]
    lines = ["path/to/cl1.fa\t%s\t%s\tinfo\t12\t10:500\t\t%s\t%s\tinfo\t9\t20:600" % (items[0] + items[1]),
             "cl2.txt\t%s\t%s\tinfo\t3\t7:300\t%s\t%s\tinfo\t2\t8:400\tAAAA" % (items[2] + items[3]),
             "cl1\t%s\t%s\tinfo\t1\t10:500\t%s\t%s\tinfo\t1\t30:700" % (items[4] + items[5]),
             "cl3"]
    path = tmp_path / "cands.sets"
    path.write_text("\n".join(lines) + "\n")
    got = sel.read_candidates(str(path), "sets")
    want = {"cl1_10_F_cl1_500": items[0], "cl1_20_F_cl1_600": items[1], "cl2_7_F_cl2_300": items[2],
            "cl2_8_F_cl2_400": items[3], "cl1_30_F_cl1_700": items[5]}
    assert list(got.items()) == list(want.items())
    _run(fa, got, str(tmp_path / "sets"), lo, hi, _backend("fake"))
    assert _files(str(tmp_path / "sets")) == restate_select(fa, want, {}, 1, lo, hi)


def _sharded(tmp_path, world, kind):
    from multiprime_b200 import primer_coverage as pc
    from tests.loopback_comm import run_shards
    backend = _backend(kind)
    fa, cands, lo, hi = make_select_case(tmp_path, 4)
    keep = {"Z": cands["Z"]}
    old = pc.S
    pc.S = 64
    try:
        _run(fa, cands, str(tmp_path / "one"), lo, hi, backend, 2, keep=keep)
        run_shards(world, lambda rank, comm: _run(fa, cands, str(tmp_path / "sharded"), lo, hi, backend, 2, comm,
                                                  keep=keep, block=2))
    finally:
        pc.S = old
    assert _files(str(tmp_path / "one")) == _files(str(tmp_path / "sharded"))


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
    return subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "primer_select.py")] + args,
                          capture_output=True, text=True, timeout=600, env=env)


@pytest.mark.parametrize("args,msg", [
    (["-k", "-1"], "-k must be >= 0"),
    (["--goal", "0"], "--goal must be in (0, 1]"),
    (["--goal", "1.5"], "--goal must be in (0, 1]"),
    (["-f", "bad"], "-f must be xls, fa or seq"),
    (["--keep", "x", "--keep-format", "sets"], "--keep-format must be xls, fa or seq"),
    (["-v", "16"], "-v must be in 0..15"),
    (["-s", "500,100"], "0 < lo <= hi"),
    (["-s", "500"], "-s takes lo,hi"),
    (["-i", "A" * 33 + ",ACGTACGTACGTACGTAC", "-f", "seq"], "primers of 1..32 bases"),
    (["-r", None], "Input (targets) file must be specified"),
])
def test_cli_errors(tmp_path, args, msg):
    fa = tmp_path / "t.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTACGT\n")
    base = {"-r": str(fa), "-i": str(tmp_path / "p.fa"), "-f": "fa", "-o": str(tmp_path / "o")}
    (tmp_path / "p.fa").write_text(">a_F\nACGTACGTACGTACGTAC\n>a_R\nTTGCATTGCATTGCATTG\n")
    for k, val in zip(args[::2], args[1::2]):
        if val is None:
            del base[k]
        else:
            base[k] = val
    res = _cli([x for kv in base.items() for x in kv])
    assert res.returncode == 1, res.stderr
    assert msg in res.stderr
    assert not os.path.exists(str(tmp_path / "o") + ".selected.tsv")


def test_too_many_pairs_refused(tmp_path):
    from multiprime_b200 import primer_select as sel
    fa = tmp_path / "t.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTACGT\n")
    cands = {"p%d" % i: ("ACGTACGTACGTACGTAC", "TTGCATTGCATTGCATTG") for i in range(sel.MAX_PAIRS + 1)}
    with pytest.raises(SystemExit, match="16385 candidate and kept pairs: at most 16384"):
        _run(str(fa), cands, str(tmp_path / "o"), 50, 500, _backend("fake"))


def test_matrix_that_cannot_be_allocated_is_refused(tmp_path, monkeypatch):
    from multiprime_b200 import _lib
    from tests import fake_pattern_cover

    class Refused(fake_pattern_cover.CoverMatrix):
        def __init__(self, ctx, n_rows, n_rec):
            raise _lib.MpbError(-3, "out of memory")
    monkeypatch.setattr(fake_pattern_cover, "CoverMatrix", Refused)
    fa, cands, lo, hi = make_select_case(tmp_path, 1)
    want = "needs %d bytes of device memory" % _lib.cover_bytes(len(cands), 31)
    with pytest.raises(SystemExit, match=want):
        _run(fa, cands, str(tmp_path / "o"), lo, hi, fake_pattern_cover)
    assert not os.path.exists(str(tmp_path / "o.selected.tsv"))


# ---------------------------------------------------------------------------------------------------------------
# torchrun
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_cli_under_torchrun(tmp_path, backend):
    """two and three ranks under torchrun write the files of one process (gloo with the ranks on cuda:0, NCCL on two
    GPUs)"""
    import torch
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    fa, cands, lo, hi = make_select_case(tmp_path, 7)
    pf = tmp_path / "cands.fa"
    pf.write_text("".join(">%s\n%s\n>R\n%s\n" % (n, f, r) for n, (f, r) in cands.items()))
    common = ["-r", fa, "-i", str(pf), "-f", "fa", "-v", "2", "-s", "%d,%d" % (lo, hi)]
    one = _cli(common + ["-o", str(tmp_path / "one")])
    assert one.returncode == 0, one.stderr[-3000:]
    assert "Selected: " in one.stdout and "Covered: " in one.stdout
    env = dict(os.environ, MPB_DIST_BACKEND=backend)
    for world in ([2] if backend == "nccl" else [2, 3]):
        tag = "w%d" % world
        res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node",
                              str(world), "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
                              os.path.join(ROOT, "scripts", "primer_select.py")] + common + ["-o", str(tmp_path / tag)],
                             capture_output=True, text=True, env=env, timeout=600)
        assert res.returncode == 0, res.stderr[-3000:]
        assert res.stdout.count("Total times") == 1
        assert _files(str(tmp_path / "one")) == _files(str(tmp_path / tag))
