"""extract_PCR_product drop-in (SURVEY.md 8f-4) against the reference script's own outputs on test_data/test.fa
(tests/golden/pcr_product.json, made by tests/golden/make_golden.py pcr): plain, degenerate (2-, 3- and 4-fold codes),
a forward primer that occurs twice in a genome, a pair without product; formats seq and fa.  Then against a
restatement of the reference's choice (str.find / str.split on each line, pinned to the same seven runs) on seeded
random FASTA files: planted and repeated sites, R sites before / inside / past F, N and lower-case stretches, and a
line longer than 65535 characters."""
import json
import os
from itertools import product as iproduct
from pathlib import Path

import numpy as np
import pytest

from tests.helpers import GOLDEN, case_alignment, load_case


def _test_fa(tmp_path):
    """test_data/test.fa rebuilt from the committed fixture of the C1 case (one line per sequence, as the original)"""
    case = load_case("c1_testfa")
    ids, seqs = case_alignment(case, "c1_testfa")
    z = np.load(os.path.join(GOLDEN, "msa_c1_testfa.npz"), allow_pickle=True)
    heads = [str(x) for x in z["headers"]]
    seqs = [list(s) for s in seqs]
    for r, c in z["n_cells"].tolist():               # the fixture stores N as a gap cell (core:453)
        seqs[r][c] = "N"
    seqs = ["".join(s) for s in seqs]
    fa = tmp_path / "test.fa"
    fa.write_text("".join(h + "\n" + s + "\n" for h, s in zip(heads, seqs)))
    return str(fa)


def _run_all(tmp_path, backend):
    from multiprime_b200 import pcr_product
    g = json.load(open(os.path.join(GOLDEN, "pcr_product.json")))
    fa = _test_fa(tmp_path)
    for run, want in g["runs"].items():
        outdir, cov = tmp_path / ("out_" + run.replace(":", "_")), tmp_path / ("cov_" + run.replace(":", "_"))
        if run.startswith("seq:"):
            f, r = g["pairs"][run[4:]]
            argv = ["-r", fa, "-i", f + "," + r, "-f", "seq", "-o", str(outdir), "-s", str(cov), "-p", "1"]
        else:
            pf = tmp_path / "primers.fa"
            pf.write_text(want["primers_fa"])
            argv = ["-r", fa, "-i", str(pf), "-f", "fa", "-o", str(outdir), "-s", str(cov), "-p", "1"]
        pcr_product.main(argv, _backend=backend)
        got = {fn: open(os.path.join(outdir, fn)).read() for fn in sorted(os.listdir(outdir))}
        assert got == want["files"], run
        assert open(cov).read() == want["coverage"], run


def test_pcr_product_host_logic(tmp_path, capsys):
    from tests import fake_device
    _run_all(tmp_path, fake_device)


@pytest.mark.gpu
def test_pcr_product_gpu(tmp_path, capsys):
    _run_all(tmp_path, None)


# ---- a restatement of the reference's choice: plain text operations on each line ------------------------------------
_DEGENERATE = {"R": "AG", "Y": "CT", "M": "AC", "K": "GT", "S": "GC", "W": "AT", "H": "ATC", "B": "GTC", "V": "GAC",
               "D": "GAT", "N": "ATGC"}                 # extract_PCR_product_V1.py:110-112, in that script's order


def _expansions(primer):
    return ["".join(t) for t in iproduct(*[_DEGENERATE.get(ch, ch) for ch in primer])]


def _rc(seq):
    return seq.translate(str.maketrans("ATGC", "TACG"))[::-1]


def _reference_product(line, f, r):
    for e in _expansions(f):
        if line.find(e) < 0:
            continue
        region = e + line.split(e)[1]                   # up to the next non-overlapping occurrence of e
        for x in _expansions(r):
            t = _rc(x)
            if region.find(t) >= 0:
                return region.split(t)[0].strip() + t
    return ""


def _reference_run(fa_text, pairs):
    """{file name: text} and the statistics text of one run of the reference on a FASTA text; pairs {name: (F, R)}"""
    keys, lines, key = [], [], None
    for raw in fa_text.splitlines(keepends=True):
        if raw.startswith(">"):
            key = raw.strip()
        else:
            keys.append(key)
            lines.append(raw)
    files, cov, covered = {}, "", set()
    for name, (f, r) in pairs.items():
        prod, non = {}, {}
        for key, line in zip(keys, lines):
            value = _reference_product(line, f, r)
            if value:
                prod[key] = value
            else:
                non[key] = line.strip()
        covered |= set(prod)
        cov += "Number of Product/non_Product, primer-F and primer-R: {}\t{}\t{}\t{}\t{}\n".format(
            name, len(prod), len(non), f, r)
        files[Path(name).with_suffix(".PCR.product.fa").name] = "".join(k + "\n" + prod[k] + "\n" for k in prod)
        files[Path(name).with_suffix(".non_PCR.product.fa").name] = "".join(k + "\n" + non[k] + "\n" for k in non)
    n_seq = int(fa_text.count("\n") / 2)
    cov += "Total number of sequences:\t{}\nCoveraged number of sequence:\t{}\nRate of coverage:\t>= {}\n".format(
        n_seq, len(covered), round(float(len(covered)) / n_seq, 2))
    return files, cov


def _primer_pairs(text):
    rows = [ln for ln in text.splitlines() if ln.strip()]
    return {rows[i].lstrip(">") + "_" + rows[i + 2].lstrip(">"): (rows[i + 1], rows[i + 3]) for i in range(0, len(rows), 4)}


def test_reference_restatement_reproduces_the_goldens(tmp_path):
    g = json.load(open(os.path.join(GOLDEN, "pcr_product.json")))
    fa = open(_test_fa(tmp_path)).read()
    for run, want in g["runs"].items():
        pairs = {"PCR_info": g["pairs"][run[4:]]} if run.startswith("seq:") else _primer_pairs(want["primers_fa"])
        files, cov = _reference_run(fa, pairs)
        assert files == want["files"], run
        assert cov == want["coverage"], run


# ---- random inputs -----------------------------------------------------------------------------------------------
RANDOM_PAIRS = [("CAGGTRACAGCTTGCA", "GGTACCTTYAGCTGAC"),          # 2-fold codes
                ("ATHGCAGTVCAGTAGC", "TTGCADCAGTGCABTT"),          # 3-fold
                ("GCANTTGACNGATC", "CCGNATGGCTANGT"),              # 4-fold
                ("CAGCAGCAGCAGCAG", "TAGGCTTACWGAGT")]             # periodic F: overlapping occurrences


def _random_fasta(seed, long_line=False):
    rng = np.random.default_rng(seed)
    pick = lambda p: "".join(rng.choice(list(_DEGENERATE.get(ch, ch))) for ch in p)
    recs = []
    for i in range(60):
        n = int(rng.integers(120, 700)) if not (long_line and i == 7) else 70_123
        s = list("".join(rng.choice(list("ACGT"), n)))

        def put(x, site):
            if 0 <= x and x + len(site) <= n:
                s[x:x + len(site)] = list(site)

        for _ in range(int(rng.integers(0, 4))):
            f, r = RANDOM_PAIRS[int(rng.integers(0, len(RANDOM_PAIRS)))]
            fe, rt = pick(f), _rc(pick(r))
            x = int(rng.integers(0, n - 60))
            kind = int(rng.integers(0, 7))
            put(x, fe)
            if kind == 0:                                   # product
                put(x + len(fe) + int(rng.integers(0, 40)), rt)
            elif kind == 1:                                 # R before F
                put(x - len(rt) - int(rng.integers(0, 20)), rt)
            elif kind == 2:                                 # R starts inside the F site
                put(x + int(rng.integers(1, len(fe))), rt)
            elif kind == 3:                                 # F again, R past the second occurrence
                y = x + len(fe) + int(rng.integers(0, 30))
                put(y, pick(f) if rng.random() < 0.5 else fe)
                put(y + len(fe) + int(rng.integers(0, 30)), rt)
            elif kind == 4:                                 # overlapping F sites
                put(x + int(rng.integers(1, len(fe))), fe)
                put(x + 2 * len(fe) + int(rng.integers(0, 30)), rt)
            elif kind == 5:                                 # R between two F sites
                put(x + len(fe) + 2, rt)
                put(x + len(fe) + len(rt) + 5, fe)
        if n > 65535:                                       # products across and past column 65535
            for f, r, x in ((RANDOM_PAIRS[0][0], RANDOM_PAIRS[0][1], 65530), (RANDOM_PAIRS[2][0], RANDOM_PAIRS[2][1], 68000)):
                put(x, pick(f))
                put(x + 400 + int(rng.integers(0, 500)), _rc(pick(r)))
        for _ in range(int(rng.integers(0, 3))):            # N and soft-masked stretches, often over a site
            x = int(rng.integers(0, n - 30))
            m = int(rng.integers(1, 30))
            s[x:x + m] = ["N"] * m if rng.random() < 0.5 else [ch.lower() for ch in s[x:x + m]]
        seq = "".join(s)
        if rng.random() < 0.15:                             # a record of two lines: each line is searched alone
            cut = int(rng.integers(1, n))
            recs.append(">seq%d\n%s\n%s\n" % (i, seq[:cut], seq[cut:]))
        else:
            recs.append(">seq%d\n%s\n" % (i, seq))
    return "".join(recs)


def _run_random(tmp_path, backend):
    from multiprime_b200 import pcr_product
    pf = tmp_path / "primers.fa"
    pf.write_text("".join(">pair%d_F\n%s\n>pair%d_R\n%s\n" % (i, f, i, r) for i, (f, r) in enumerate(RANDOM_PAIRS)))
    pairs = _primer_pairs(pf.read_text())
    n_products = 0
    for seed, long_line in ((1, False), (2, False), (3, True)):
        fa = tmp_path / ("in%d.fa" % seed)
        fa.write_text(_random_fasta(seed, long_line))
        outdir, cov = tmp_path / ("out%d" % seed), tmp_path / ("cov%d" % seed)
        pcr_product.main(["-r", str(fa), "-i", str(pf), "-f", "fa", "-o", str(outdir), "-s", str(cov), "-p", "1"],
                         _backend=backend)
        want_files, want_cov = _reference_run(fa.read_text(), pairs)
        got = {fn: open(os.path.join(outdir, fn)).read() for fn in sorted(os.listdir(outdir))}
        assert got == want_files, seed
        assert open(cov).read() == want_cov, seed
        n_products += sum(v.count(">") for k, v in want_files.items() if k.endswith(".PCR.product.fa"))
    assert n_products > 40


def test_pcr_product_random_host_logic(tmp_path, capsys):
    from tests import fake_device
    _run_random(tmp_path, fake_device)


@pytest.mark.gpu
def test_pcr_product_random_gpu(tmp_path, capsys):
    _run_random(tmp_path, None)
