"""primer_select --cross / --background end to end against a plain-Python restatement: test_primer_select's
restate_select extended with test_primer_specificity's restate_groups (str slicing over every (i, j)) for the cross
products of each take and the own products on the background; on the CPU double and on the GPU, in one rank,
thread-sharded and under torchrun.  On the GPU also the invariant the flags promise, re-checked by primer_specificity on
selected.fa."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.test_primer_coverage import _free_port, rc, restate
from tests.test_primer_select import THRESHOLD, _files, make_select_case
from tests.test_primer_specificity import restate_groups

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _backend(kind):
    if kind == "gpu":
        from multiprime_b200 import _lib
        return _lib
    from tests import fake_site_list
    return fake_site_list


# ---------------------------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------------------------
def _products(fasta_text, rows, v, lo, hi):
    """{(i, j)} with a product on some record of fasta_text; primer 2q = F of row q, 2q + 1 = R"""
    pairs = {str(q): (f, r) for q, (_, f, r) in enumerate(rows)}
    _, _, _, groups = restate_groups(fasta_text, pairs, v, "1,2,-1", lo, hi)
    return {(i, j) for _, i, j in groups}


def restate_select(fa, cands, keep, v, lo, hi, max_pairs=0, goal=1.0, cross=False, background=None):
    """(selected.tsv, candidates.tsv, selected.fa) as text; cands / keep: {name: (F, R)}"""
    from oracle.dimer_oracle import find_dimers
    rows = [(n, f.strip().upper(), r.strip().upper()) for n, (f, r) in keep.items()]
    rows += [(n, f.strip().upper(), r.strip().upper()) for n, (f, r) in cands.items() if n not in keep]
    row_of = {n: i for i, (n, _, _) in enumerate(rows)}
    n_keep = len(keep)
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
    dimers = {frozenset((d[1], d[8])) for d in find_dimers({s: ">s%d" % k for k, s in enumerate(seqs)}, THRESHOLD)}

    def conflict(a, b):
        return a != b and any(sa != sb and frozenset((sa, sb)) in dimers for sa in rows[a][1:] for sb in rows[b][1:])

    def seq(i):
        return rows[i // 2][1 + i % 2]

    prods = _products(open(fa).read(), rows, v, lo, hi) if cross else set()
    bg_prods = _products(open(background).read(), rows, v, lo, hi) if background else set()
    if cross:
        prods |= bg_prods
    excluded = {}
    for c in range(n_keep, len(rows)):
        if any(i // 2 == c and j // 2 == c for i, j in bg_prods):
            excluded[c] = (0, None, "off-target")
    covered, covered_p = set(), set()
    taken = []

    def is_cross(q, c):
        intended = set()
        for t in [t[0] for t in taken] + [c]:
            intended |= {(rows[t][1], rows[t][2]), (rows[t][2], rows[t][1])}
        for i, j in prods:
            if {i // 2, j // 2} == {q, c} and seq(i) != seq(j) and (seq(i), seq(j)) not in intended:
                return True
        return False

    def take(q, step):
        new, newp = A[q] - covered, P[q] - covered_p
        covered.update(A[q])
        covered_p.update(P[q])
        taken.append((q, step, len(new), len(newp), len(covered), len(covered_p)))
        for c in range(n_keep, len(rows)):
            if c not in excluded and all(c != t[0] for t in taken) and conflict(q, c):
                excluded[c] = (step, q, "dimer")
        for c in range(n_keep, len(rows)):
            if cross and c not in excluded and all(c != t[0] for t in taken) and is_cross(q, c):
                excluded[c] = (step, q, "cross")

    for q in range(n_keep):
        take(q, 0)
    step = 0
    while not (max_pairs and step >= max_pairs) and len(covered) / n_targets < goal:
        best = None
        for c in range(n_keep, len(rows)):
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
        if q < n_keep:
            st = ("kept", "0", "-")
        elif q in step_of:
            st = ("selected", str(step_of[q]), "-")
        elif q in excluded:
            s, by, status = excluded[q]
            st = (status, str(s), "-" if by is None else rows[by][0])
        else:
            st = ("open", "-", "-")
        cand.append("%s\t%s\t%s\t%d\t%d\t%s\t%s\t%s\n" % ((name,) + rows[q][1:] + (len(A[q]), len(P[q])) + st))
    return "".join(sel), "".join(cand), "".join(fasta)


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def make_specific_case(tmp_path, seed):
    """(targets, background, candidates, lo, hi): test_primer_select's case plus
      bgcross    F random, R = RC of a site that only the background holds, after X's F: a cross product of X that
                 exists only on the background;
      shareF     X's F with another R: (X:F, shareF:R) is intended, not cross;
      offlo      its own (F, R) product on the background is exactly lo long and ends where its record ends;
      offhi      the same at exactly hi;
      offself    its F binds both strands of a background record, an (F, F) product;
      tight      its R site starts right where X's F site ends on a background record (y = x + L_i): a 40-base
                 cross product of X, inside -s only when lo <= 40.
    Z stays a dimer of X and is also a cross product of X (Z:F at 100, X:R at 800)."""
    fa, cands, lo, hi = make_select_case(tmp_path, seed)
    rng = np.random.default_rng(seed + 1000)
    root = "".join(np.random.default_rng(seed).choice(list("ACGT"), 1400))

    def rand(n):
        return "".join(rng.choice(list("ACGT"), n))
    xf = root[300:320]
    site = rand(20)
    cands["bgcross"] = (rand(20), rc(site))
    cands["shareF"] = (xf, rc(root[700:720]))
    f_lo, r_lo, f_hi, r_hi, f_self = rand(20), rand(20), rand(20), rand(20), rand(20)
    cands["offlo"] = (f_lo, rc(r_lo))
    cands["offhi"] = (f_hi, rc(r_hi))
    cands["offself"] = (f_self, rc(rand(20)))
    tight = rand(20)
    cands["tight"] = (rand(20), rc(tight))
    bg = [("bg_cross", rand(50) + xf + rand(300) + site + rand(50)),
          ("bg_lo", rand(30) + f_lo + rand(lo - 40) + r_lo),
          ("bg_hi", f_hi + rand(hi - 40) + r_hi + rand(7)),
          ("bg_self", rand(10) + f_self + rand(200) + rc(f_self) + rand(10)),
          ("bg_tight", rand(40) + xf + tight + rand(3)),
          ("bg_random", rand(3000))]
    path = tmp_path / ("background%d.fa" % seed)
    path.write_text("".join(">%s\n%s\n" % (n, s) for n, s in bg))
    return fa, str(path), cands, lo, hi


def _run(fa, cands, out, lo, hi, backend, v=1, comm=None, keep=None, **kw):
    from multiprime_b200 import primer_select as sel
    return sel.run(fa, cands, out, v, "1,2,-1", (lo, hi), kw.get("max_pairs", 0), kw.get("goal", 1.0), THRESHOLD, keep,
                   kw.get("cross", False), kw.get("background"), comm=comm, _backend=backend, _block=kw.get("block", 0))


FLAGS = [dict(cross=True), dict(bg=True), dict(cross=True, bg=True), dict(cross=True, bg=True, keep=["X"]),
         dict(cross=True, keep=["X", "W"], block=3), dict(cross=True, bg=True, max_pairs=1),
         dict(cross=True, bg=True, goal=0.5, block=1), dict(bg=True, keep=["offlo"]), dict(cross=True, bg=True, lo=40)]


def _check(tmp_path, kind, flags, seed=1, v=1):
    kw = dict(flags)
    fa, bgfa, cands, lo, hi = make_specific_case(tmp_path, seed)
    lo = kw.pop("lo", lo)
    if kw.pop("bg", False):
        kw["background"] = bgfa
    keep = {k: cands[k] for k in kw.pop("keep", [])}
    out = str(tmp_path / kind)
    _run(fa, cands, out, lo, hi, _backend(kind), v, keep=keep, **kw)
    want = restate_select(fa, cands, keep, v, lo, hi, kw.get("max_pairs", 0), kw.get("goal", 1.0),
                          kw.get("cross", False), kw.get("background"))
    got = _files(out)
    assert got == want
    return {r.split("\t")[0]: r.split("\t")[5:] for r in got[1].splitlines()[1:]}


def _assert_case_covers(flags, status):
    bg, cross, keep = flags.get("bg"), flags.get("cross"), flags.get("keep", [])
    if bg:
        for name in ("offlo", "offhi", "offself"):
            assert status[name] == (["kept", "0", "-"] if name in keep else ["off-target", "0", "-"]), name
    else:
        assert "off-target" not in {s[0] for s in status.values()}
    if not cross:
        assert "cross" not in {s[0] for s in status.values()}
    if cross and keep[:1] == ["X"]:
        assert status["Z"] == ["dimer", "0", "X"]
        assert status["shareF"][:2] != ["cross", "0"]
        assert status["bgcross"] == (["cross", "0", "X"] if bg else ["open", "-", "-"])
        if flags.get("lo") == 40:
            assert status["tight"] == ["cross", "0", "X"]


@pytest.mark.parametrize("flags", range(len(FLAGS)))
def test_flags_match_restatement_fake(tmp_path, flags):
    _assert_case_covers(FLAGS[flags], _check(tmp_path, "fake", FLAGS[flags]))


@pytest.mark.gpu
@pytest.mark.parametrize("flags", range(len(FLAGS)))
def test_flags_match_restatement_gpu(tmp_path, flags):
    _assert_case_covers(FLAGS[flags], _check(tmp_path, "gpu", FLAGS[flags]))


def test_tight_and_exact_ends_fake(tmp_path):
    """with X kept, lo = 40 and both flags: the y = x + L_i product excludes tight, and bgcross is excluded by the
    background alone"""
    flags = dict(cross=True, bg=True, keep=["X"], lo=40)
    _assert_case_covers(flags, _check(tmp_path, "fake", flags))


@pytest.mark.gpu
def test_tight_and_exact_ends_gpu(tmp_path):
    flags = dict(cross=True, bg=True, keep=["X"], lo=40)
    _assert_case_covers(flags, _check(tmp_path, "gpu", flags))


def test_without_flags_matches_plain_select_fake(tmp_path):
    """no flag: the files of test_primer_select's restatement, the new candidates included"""
    from tests.test_primer_select import restate_select as plain
    fa, _, cands, lo, hi = make_specific_case(tmp_path, 3)
    out = str(tmp_path / "plain")
    _run(fa, cands, out, lo, hi, _backend("fake"))
    assert _files(out) == plain(fa, cands, {}, 1, lo, hi)


def _sharded(tmp_path, world, kind):
    from multiprime_b200 import primer_coverage as pc
    from tests.loopback_comm import run_shards
    backend = _backend(kind)
    fa, bgfa, cands, lo, hi = make_specific_case(tmp_path, 4)
    keep = {"Z": cands["Z"]}
    old = pc.S
    pc.S = 64
    try:
        _run(fa, cands, str(tmp_path / "one"), lo, hi, backend, 2, keep=keep, cross=True, background=bgfa)
        run_shards(world, lambda rank, comm: _run(fa, cands, str(tmp_path / "sharded"), lo, hi, backend, 2, comm,
                                                  keep=keep, block=2, cross=True, background=bgfa))
        want = restate_select(fa, cands, keep, 2, lo, hi, cross=True, background=bgfa)
    finally:
        pc.S = old
    assert _files(str(tmp_path / "one")) == _files(str(tmp_path / "sharded")) == want


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_threads_write_the_same_files_fake(tmp_path, world):
    _sharded(tmp_path, world, "fake")


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_threads_write_the_same_files_gpu(tmp_path, world):
    _sharded(tmp_path, world, "gpu")


# ---------------------------------------------------------------------------------------------------------------
# the invariant, re-checked by primer_specificity on selected.fa
# ---------------------------------------------------------------------------------------------------------------
def _spec_rows(fa, selected_fa, out, lo, hi, v):
    from multiprime_b200 import _lib
    from multiprime_b200 import primer_specificity as ps
    from multiprime_b200.pcr_product import parse_primers
    ps.run(fa, parse_primers(selected_fa, "fa"), out, v, "1,2,-1", (lo, hi), _backend=_lib)
    return [r.split("\t") for r in open(out + ".specificity.tsv").read().splitlines()[1:-1]]


def _pair(primer):
    """the selected pair of a primer read back from selected.fa: parse_primers names it <name>:F_<name>:R"""
    return primer.rsplit(":", 1)[0].split(":F_")[0]


def _invariant(tmp_path, kind, seed, keep):
    """--cross: no cross combination between two selected pairs unless both are kept; with --background as well, no
    product on the background of any combination that involves a pair taken at step >= 1 (the case shares no primer
    sequence between two pairs once shareF, pair1_copy and W_copy are dropped)"""
    from multiprime_b200 import primer_specificity as ps
    from multiprime_b200.pcr_product import parse_primers
    fa, bgfa, cands, lo, hi = make_specific_case(tmp_path, seed)
    for name in ("shareF", "pair1_copy", "W_copy"):
        cands.pop(name)
    keep = {k: cands[k] for k in keep}
    out = str(tmp_path / "sel")
    _run(fa, cands, out, lo, hi, _backend(kind), 2, keep=keep, cross=True, background=bgfa)
    sel = [r.split("\t") for r in open(out + ".selected.tsv").read().splitlines()[1:]]
    late = {r[1] for r in sel if int(r[0]) >= 1}
    assert late
    spec = _lib_backend(kind)
    rows = {}
    for tag, ref in (("t", fa), ("b", bgfa)):
        ps.run(ref, parse_primers(out + ".selected.fa", "fa"), str(tmp_path / tag), 2, "1,2,-1", (lo, hi),
               _backend=spec)
        rows[tag] = [r.split("\t") for r in open(str(tmp_path / tag) + ".specificity.tsv").read().splitlines()[1:-1]]
    for left, right, klass, *_ in rows["t"]:
        if klass == "cross":
            assert _pair(left) in keep and _pair(right) in keep, (left, right)
    for left, right, *_ in rows["b"]:
        assert _pair(left) not in late and _pair(right) not in late, (left, right)
    return late


def _lib_backend(kind):
    if kind == "gpu":
        from multiprime_b200 import _lib
        return _lib
    from tests import fake_pattern_products
    return fake_pattern_products


INVARIANT = [(1, []), (5, []), (1, ["W"]), (5, ["W"])]


@pytest.mark.parametrize("case", range(len(INVARIANT)))
def test_selected_set_has_no_cross_or_background_product_fake(tmp_path, case):
    _invariant(tmp_path, "fake", *INVARIANT[case])


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(INVARIANT)))
def test_selected_set_has_no_cross_or_background_product_gpu(tmp_path, case):
    _invariant(tmp_path, "gpu", *INVARIANT[case])


# ---------------------------------------------------------------------------------------------------------------
# CLI
# ---------------------------------------------------------------------------------------------------------------
def _cli(args, env=None):
    return subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "primer_select.py")] + args,
                          capture_output=True, text=True, timeout=600, env=env)


def test_site_list_that_cannot_be_allocated_is_refused(tmp_path, monkeypatch):
    from multiprime_b200 import _lib
    from tests import fake_site_list

    class Refused(fake_site_list.SiteList):
        def seal(self):
            raise _lib.MpbError(-3, "the site list's sort buffer of 12 sites needs 96 bytes of device memory")
    monkeypatch.setattr(fake_site_list, "SiteList", Refused)
    fa, _, cands, lo, hi = make_specific_case(tmp_path, 1)
    with pytest.raises(SystemExit, match="Error: .*needs 96 bytes of device memory"):
        _run(fa, cands, str(tmp_path / "o"), lo, hi, fake_site_list, cross=True)
    assert not os.path.exists(str(tmp_path / "o.selected.tsv"))


@pytest.mark.gpu
@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_cli_under_torchrun(tmp_path, backend):
    """two and three ranks under torchrun with --cross and --background write the files of one process"""
    import torch
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    fa, bgfa, cands, lo, hi = make_specific_case(tmp_path, 7)
    pf = tmp_path / "cands.fa"
    pf.write_text("".join(">%s\n%s\n>R\n%s\n" % (n, f, r) for n, (f, r) in cands.items()))
    common = ["-r", fa, "-i", str(pf), "-f", "fa", "-v", "2", "-s", "%d,%d" % (lo, hi), "--cross", "--background", bgfa]
    one = _cli(common + ["-o", str(tmp_path / "one")])
    assert one.returncode == 0, one.stderr[-3000:]
    assert "\tcross\t" in _files(str(tmp_path / "one"))[1] and "\toff-target\t0\t-\n" in _files(str(tmp_path / "one"))[1]
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
