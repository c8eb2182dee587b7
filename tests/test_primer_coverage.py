"""primer_coverage end to end against a plain-Python restatement of its semantics (str slicing on both strands, no numpy):
on the CPU double and on the GPU, in one rank and sequence-sharded, plus its CLI errors."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IUPAC = {"A": "A", "C": "C", "G": "G", "T": "T", "R": "AG", "Y": "CT", "M": "AC", "K": "GT", "S": "CG", "W": "AT",
         "H": "ACT", "B": "CGT", "V": "ACG", "D": "AGT", "N": "ACGT"}
COMP = {"A": "T", "C": "G", "G": "C", "T": "A"}


# ---------------------------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------------------------
def read_records(text):
    recs = []
    for line in text.replace("\r", "").split("\n"):
        if line.startswith(">"):
            words = line[1:].split()
            recs.append([words[0] if words else "", []])
        elif recs:
            recs[-1][1].append(line)
    out = []
    for name, lines in recs:
        seq = []
        for ch in "".join(lines).upper():
            if ch in "-.":
                continue
            seq.append("T" if ch == "U" else ch if ch in IUPAC else "N")
        out.append((name, "".join(seq)))
    return out


def rc(seq):
    return "".join(COMP.get(ch, "N") for ch in reversed(seq))


def strict_positions(coordinate, k):
    f, r = set(), set()
    for tok in coordinate.split(","):
        y = int(tok)
        fi, ri = (y, k - y) if y > 0 else (k + y + 1, -y + 1)
        if 0 <= fi < k:
            f.add(fi)
        if 0 <= ri < k:
            r.add(ri)
    return f, r


def find(seq, primer, strict, v):
    """[(x, mismatches)] of the primer on seq"""
    out = []
    L = len(primer)
    for x in range(len(seq) - L + 1):
        mis = 0
        for i, ch in enumerate(primer):
            c = seq[x + i]
            if c not in "ACGT" or c not in IUPAC.get(ch, ""):
                mis += 1
                if i in strict or mis > v:
                    mis = -1
                    break
        if mis >= 0:
            out.append((x, mis))
    return out


def restate(fasta_text, pairs, v, coordinate, lo, hi):
    """(amplicons.tsv, coverage.tsv) as text"""
    recs = read_records(fasta_text)
    amp = ["#Pair\tTarget\tStrand\tStart\tEnd\tLength\tF_mismatches\tR_mismatches\n"]
    cov = ["#Pair\tPrimer_F\tPrimer_R\tAmplified\tPerfect\tTotal\tCoverage\n"]
    any_amp, any_perf = set(), set()
    for name, (f, r) in pairs.items():
        f, r = f.upper(), r.upper()
        lf, lr = len(f), len(r)
        fs, _ = strict_positions(coordinate, lf)
        _, rs = strict_positions(coordinate, lr)
        rs_r = {lr - 1 - j for j in rs}              # rmask is over RC(R): as positions of R itself
        n_amp = n_perf = 0
        for ti, (tname, seq) in enumerate(recs):
            n = len(seq)
            best = None
            f_fwd, f_rev = find(seq, f, fs, v), find(rc(seq), f, fs, v)
            r_fwd, r_rev = find(seq, r, rs_r, v), find(rc(seq), r, rs_r, v)
            # + strand: F on the record, R on its reverse complement
            for x, mf in f_fwd:
                for q, mr in r_rev:
                    y = n - q - lr
                    length = y + lr - x
                    if y >= x + lf and lo <= length <= hi:
                        key = (mf + mr, length, 0, x, mf, mr)
                        best = key if best is None or key < best else best
            # - strand: R on the record, F on its reverse complement
            for x, mr in r_fwd:
                for q, mf in f_rev:
                    y = n - q - lf
                    length = y + lf - x
                    if y >= x + lr and lo <= length <= hi:
                        key = (mf + mr, length, 1, x, mf, mr)
                        best = key if best is None or key < best else best
            if best is None:
                continue
            tot, length, strand, x, mf, mr = best
            amp.append("%s\t%s\t%s\t%d\t%d\t%d\t%d\t%d\n" % (name, tname, "+-"[strand], x, x + length, length, mf, mr))
            n_amp += 1
            any_amp.add(ti)
            if tot == 0:
                n_perf += 1
                any_perf.add(ti)
        cov.append("%s\t%s\t%s\t%d\t%d\t%d\t%s\n" % (name, f, r, n_amp, n_perf, len(recs), round(n_amp / len(recs), 4)))
    cov.append("ALL\t-\t-\t%d\t%d\t%d\t%s\n" % (len(any_amp), len(any_perf), len(recs),
                                                round(len(any_amp) / len(recs), 4)))
    return "".join(amp), "".join(cov)


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def make_case(tmp_path, seed):
    """(fasta path, primer file path, lo, hi): targets cut from one root with point mutations, indels, N runs,
    IUPAC cells, other characters, gaps, U, lower case and multi-line records, half of them reverse-complemented; a record of several root
    copies (longer than the row stride, ties between equal amplicons, + against -); two records that meet in the middle
    of a primer site; products of exactly lo and hi"""
    rng = np.random.default_rng(seed)
    root = "".join(rng.choice(list("ACGT"), 1400))
    pairs, prods = {}, []
    for q, (a, b) in enumerate(((60, 700), (210, 1100), (400, 560))):
        lf, lr = 20 + q, 19 + 2 * q
        f = list(root[a:a + lf])
        f[5] = {"A": "R", "G": "R", "C": "Y", "T": "Y"}[f[5]]
        r = rc(root[b:b + lr])
        pairs["pair%d" % q] = ("".join(f), r)
        prods.append(b + lr - a)
    lo, hi = min(prods), max(prods)

    def mutate(s):
        s = list(s)
        for _ in range(int(rng.integers(0, 12))):
            i = int(rng.integers(0, len(s)))
            kind = rng.random()
            if kind < 0.6:
                s[i] = str(rng.choice(list("ACGT")))
            elif kind < 0.75:
                s.insert(i, str(rng.choice(list("ACGT"))))
            elif kind < 0.9:
                del s[i]
            else:
                s[i] = str(rng.choice(list("NRYKMSWBDHVX*")))
        if rng.random() < 0.2:
            i = int(rng.integers(0, len(s) - 10))
            s[i:i + int(rng.integers(2, 9))] = ["N"] * int(rng.integers(2, 9))
        return "".join(s)

    recs = []
    for t in range(26):
        s = mutate(root)
        a = int(rng.integers(0, 120))
        s = s[a:len(s) - int(rng.integers(0, 120))]
        if t % 2:
            s = rc(s)
        recs.append(("t%02d some description" % t, s))
    recs.append(("exact", root))
    recs.append(("copies", root + root + root[:900] + rc(root)))
    recs.append(("left_half", root[:90] + root[200:]))
    recs.append(("cut_a", "ACGT" * 5 + root[60:60 + 17]))                   # 17 bases of F, then the record ends
    recs.append(("cut_b", root[60 + 17:900]))
    lines = []
    for name, s in recs:
        s = "".join(ch.lower() if rng.random() < 0.1 else ch for ch in s)
        s = "".join(("U" if ch == "T" else "u" if ch == "t" else ch) if rng.random() < 0.05 else ch for ch in s)
        s = "".join(ch + ("-" if rng.random() < 0.01 else "." if rng.random() < 0.005 else "") for ch in s)
        step = int(rng.choice([60, 80, 10_000]))
        lines.append(">" + name)
        lines += [s[i:i + step] for i in range(0, len(s), step)]
    fa = tmp_path / ("targets%d.fa" % seed)
    fa.write_text("\n".join(lines) + "\n")
    pf = tmp_path / ("primers%d.fa" % seed)
    pf.write_text("".join(">%s_F\n%s\n>%s_R\n%s\n" % (n, f, n, r) for n, (f, r) in pairs.items()))
    return str(fa), str(pf), lo, hi


def _run_tool(fa, pf, out, v, lo, hi, backend, comm=None):
    from multiprime_b200 import primer_coverage as pc
    from multiprime_b200.pcr_product import parse_primers
    pc.run(fa, parse_primers(pf, "fa"), out, v, "1,2,-1", (lo, hi), comm=comm, _backend=backend)


def _check(tmp_path, fa, pf, lo, hi, v, backend, tag):
    from multiprime_b200.pcr_product import parse_primers
    out = str(tmp_path / tag)
    _run_tool(fa, pf, out, v, lo, hi, backend)
    want_amp, want_cov = restate(open(fa).read(), parse_primers(pf, "fa"), v, "1,2,-1", lo, hi)
    assert open(out + ".amplicons.tsv").read() == want_amp
    assert open(out + ".coverage.tsv").read() == want_cov
    return want_amp


def _assert_case_covers(amp, lo, hi):
    rows = [ln.split("\t") for ln in amp.splitlines()[1:]]
    lengths = {int(r[5]) for r in rows}
    assert lo in lengths and hi in lengths
    assert {r[2] for r in rows} == {"+", "-"}
    assert any(int(r[6]) + int(r[7]) > 0 for r in rows)
    assert not any(r[1] in ("cut_a", "cut_b") and r[0] == "pair0" for r in rows)


@pytest.mark.parametrize("stride", [64, None])
@pytest.mark.parametrize("v", [1, 3])
def test_tool_matches_restatement_fake(tmp_path, monkeypatch, stride, v):
    from multiprime_b200 import primer_coverage as pc
    from tests import fake_pattern_sites
    if stride:
        monkeypatch.setattr(pc, "S", stride)
    fa, pf, lo, hi = make_case(tmp_path, seed=v)
    amp = _check(tmp_path, fa, pf, lo, hi, v, fake_pattern_sites, "fake")
    _assert_case_covers(amp, lo, hi)


@pytest.mark.gpu
@pytest.mark.parametrize("stride", [64, None])
@pytest.mark.parametrize("v", [0, 1, 3])
def test_tool_matches_restatement_gpu(tmp_path, monkeypatch, stride, v):
    from multiprime_b200 import _lib
    from multiprime_b200 import primer_coverage as pc
    if stride:
        monkeypatch.setattr(pc, "S", stride)
    fa, pf, lo, hi = make_case(tmp_path, seed=v + 10)
    _check(tmp_path, fa, pf, lo, hi, v, _lib, "gpu")


def test_straddling_site_is_found_and_dropped(tmp_path):
    """the search reports the F site that runs from the end of cut_a into the gap cells after it (3 mismatches), and
    the host drops it because it leaves the record"""
    from multiprime_b200 import primer_coverage as pc
    from multiprime_b200.pcr_product import parse_primers
    from tests import fake_pattern_sites
    fa, pf, lo, hi = make_case(tmp_path, seed=3)
    t = pc.read_targets(fa)
    panel = pc.Panel(parse_primers(pf, "fa"), "1,2,-1")
    rows, width, starts = pc.layout(t, panel.lmax)
    msa = fake_pattern_sites.Msa(None, rows, len(rows), width, row_bytes=rows.shape[1])
    hp, hr, hx, hm = msa.pattern_sites(panel.allow, panel.plen, panel.strict, 3)
    cut = t.names.index("cut_a")
    g = np.asarray(hr, np.int64) * pc.S + hx
    raw = (hp == 0) & (g == starts[cut] + t.lens[cut] - 17)
    assert raw.sum() == 1
    kept = pc.stream_sites(np.asarray(hp, np.int64), np.asarray(hr, np.int64), np.asarray(hx, np.int64),
                           np.asarray(hm, np.int64), panel.plen.astype(np.int64), starts, t.lens)
    assert not ((kept[0] == 0) & (kept[1] == cut)).any()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_threads_write_the_same_files(tmp_path, monkeypatch, world):
    from multiprime_b200 import primer_coverage as pc
    from tests import fake_pattern_sites
    from tests.loopback_comm import run_shards
    monkeypatch.setattr(pc, "S", 64)
    fa, pf, lo, hi = make_case(tmp_path, seed=5)
    _run_tool(fa, pf, str(tmp_path / "one"), 2, lo, hi, fake_pattern_sites)
    run_shards(world, lambda rank, comm: _run_tool(fa, pf, str(tmp_path / "sharded"), 2, lo, hi, fake_pattern_sites, comm))
    for ext in (".amplicons.tsv", ".coverage.tsv"):
        assert open(str(tmp_path / "one") + ext).read() == open(str(tmp_path / "sharded") + ext).read()


# ---------------------------------------------------------------------------------------------------------------
# CLI
# ---------------------------------------------------------------------------------------------------------------
def _cli(args, env=None):
    return subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "primer_coverage.py")] + args,
                          capture_output=True, text=True, timeout=300, env=env)


@pytest.mark.parametrize("args,msg", [
    (["-v", "16"], "-v must be in 0..15"),
    (["-i", "A" * 33 + ",ACGTACGTACGTACGTAC", "-f", "seq"], "primers of 1..32 bases"),
    (["-s", "500,100"], "0 < lo <= hi"),
    (["-r", None], "Input (targets) file must be specified"),
    (["-v", "3", "-i", "ACG,ACGTACGTACGTACGTAC", "-f", "seq"], "not smaller than the shortest primer"),
])
def test_cli_errors(tmp_path, args, msg):
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
    assert not os.path.exists(str(tmp_path / "o") + ".coverage.tsv")


# ---------------------------------------------------------------------------------------------------------------
# torchrun
# ---------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_cli_under_torchrun(tmp_path, backend):
    """two ranks under torchrun write the files of one process: gloo with both ranks on cuda:0, NCCL on two GPUs"""
    import torch
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    fa, pf, lo, hi = make_case(tmp_path, seed=7)
    common = ["-r", fa, "-i", pf, "-f", "fa", "-v", "2", "-s", "%d,%d" % (lo, hi)]
    one = _cli(common + ["-o", str(tmp_path / "one")])
    assert one.returncode == 0, one.stderr[-3000:]
    env = dict(os.environ, MPB_DIST_BACKEND=backend)
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                          "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
                          os.path.join(ROOT, "scripts", "primer_coverage.py")] + common + ["-o", str(tmp_path / "two")],
                         capture_output=True, text=True, env=env, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    assert res.stdout.count("Total times") == 1
    for ext in (".amplicons.tsv", ".coverage.tsv"):
        assert open(str(tmp_path / "one") + ext).read() == open(str(tmp_path / "two") + ext).read()
