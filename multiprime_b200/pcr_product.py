"""Drop-in for scripts/extract_PCR_product.py (extract_PCR_product_V1.py): exact in-silico PCR of (degenerate) primer pairs
against a raw FASTA — the coverage validation of the pipeline, done exhaustively (SURVEY.md 8f-4).

Same flags (-r -i -f -o -p -s) and output files: <out>/<pair>.PCR.product.fa, <out>/<pair>.non_PCR.product.fa and the
statistics file (appended to, as the reference does).  The reference searches every expansion of the forward primer as a
plain string in every sequence line (extract_PCR_product_V1.py:189-216); here ONE GPU pass over every position of every
sequence finds all occurrences of all expansions of all primers (mpb_pattern_hits: the scan kernel with the window start
as a free variable), and the host only replays the reference's choice among the few hits:

    for each expansion e of F, in product order, that occurs in the line:
        Product = line[first occurrence of e : second (non-overlapping) occurrence of e, or end of line]
        for each expansion r of R, in product order, whose reverse complement occurs in Product:
            product = Product[: first occurrence of RC(r)] .strip() + RC(r);  stop
        stop at the first e that yields a product

Rows of the output are in primer order (the reference's order depends on process scheduling when -p > 1).
Limits: primers longer than 32 bases are not supported."""
from __future__ import annotations

import os
import sys
import time
from itertools import product as iproduct
from optparse import OptionParser
from pathlib import Path

import numpy as np

from . import _lib
from .core import pack4

# extract_PCR_product_V1.py:110-112 (N included; this script's own order)
DEGENERATE_BASE = {"R": ["A", "G"], "Y": ["C", "T"], "M": ["A", "C"], "K": ["G", "T"], "S": ["G", "C"], "W": ["A", "T"],
                   "H": ["A", "T", "C"], "B": ["G", "T", "C"], "V": ["G", "A", "C"], "D": ["G", "A", "T"],
                   "N": ["A", "T", "G", "C"]}
_BASE_BIT = {"A": 1, "C": 2, "G": 4, "T": 8}
_TRANS = str.maketrans("ATGC", "TACG")


def RC(seq: str) -> str:
    return seq.translate(_TRANS)[::-1]


def argsParse(argv=None):
    parser = OptionParser('Usage: %prog -r [input] -i [primerF,primerR] -f [format] -o [output]', version="%prog 0.0.2")
    parser.add_option('-r', '--ref', dest='ref', help='reference file: template fasta or reference fasta.')
    parser.add_option('-i', '--input', dest='input',
                      help='Primer file. One of: final_maxprimers_set.xls, primer.fa, primer_F,primer_R.')
    parser.add_option('-f', '--format', dest='format', help='Format of primer file: xls or fa or seq.')
    parser.add_option('-o', '--out', dest='out', default="PCR_product", help='Output_dir. default: PCR_product.')
    parser.add_option('-p', '--process', dest='process', default="10", type="int",
                      help='Number of process to launch (accepted; the search runs on the GPU). default: 10.')
    parser.add_option('-s', '--stast', dest='stast', default="Coverage.xls",
                      help='Stast information: number of coverage and total. default: Coverage.xls')
    parser.add_option('--device', dest='device', default=0, type="int", help="(hidden) CUDA device")
    args = sys.argv[1:] if argv is None else argv
    (options, rest) = parser.parse_args(args)
    if len(args) == 0:
        parser.print_help()
        sys.exit(1)
    for value, msg in ((options.ref, "Input (reference) file must be specified !!!"),
                       (options.input, "Primer file or sequence must be specified !!!"),
                       (options.format, "Primer file format must be specified !!!"),
                       (options.out, "No output file provided !!!")):
        if value is None:
            parser.print_help()
            print(msg)
            sys.exit(1)
    return options


def expansion_order(primer: str):
    """the expansions of a primer in the order of extract_PCR_product_V1.py:169-187 (leftmost position slowest)"""
    alts = [DEGENERATE_BASE.get(ch, [ch]) for ch in primer]
    return ["".join(t) for t in iproduct(*alts)]


def allow_of(primer: str):
    """allowed-base masks of a primer: bit i of mask b set when base b (A,C,G,T) is allowed at position i; characters
    outside the IUPAC alphabet allow nothing there (they cannot occur in an expansion either)"""
    allow = [0, 0, 0, 0]
    for i, ch in enumerate(primer):
        for base in DEGENERATE_BASE.get(ch, [ch]):
            if base in _BASE_BIT:
                allow["ACGT".index(base)] |= 1 << i
    return allow


def parse_primers(primer_file, file_format):
    """extract_PCR_product_V1.py:141-167: {pair name: [primer_F, primer_R]} from a final_maxprimers_set.xls (xls), a
    four-line-per-pair FASTA (fa) or "F,R" (seq)"""
    res = {}
    if file_format == "seq":
        primers = primer_file.split(",")
        res["PCR_info"] = [primers[0], primers[1]]
        return res
    with open(primer_file, "r") as f:
        if file_format == "xls":
            for line in f:
                if line.startswith("#"):
                    continue
                i = line.strip().split("\t")
                cluster_id = i[0].split("/")[-1].split(".")[0]
                start, stop = i[6].split(":")[0], i[6].split(":")[1]
                res[cluster_id + "_" + str(start) + "_F_" + cluster_id + "_" + str(stop)] = [i[2], i[3]]
        elif file_format == "fa":
            rows = [ln.rstrip("\n") for ln in f if ln.strip() != ""]      # pandas.read_table skips blank lines
            for idx, row in enumerate(rows):
                if idx % 4 == 0:
                    primer_f_info = row.lstrip(">")
                elif idx % 4 == 1:
                    primer_f = row
                elif idx % 4 == 2:
                    key = primer_f_info + "_" + row.lstrip(">")
                else:
                    res[key] = [primer_f, row]
    return res


class Product(object):
    """extract_PCR_product_V1.py:123-133 constructor arguments"""

    def __init__(self, primer_file="", output_file="", ref_file="", file_format="fa", coverage="", nproc=10, device=0,
                 _backend=None):
        self.nproc = nproc
        self.primers_file = primer_file
        self.ref_file = ref_file
        self.output_file = Path(output_file)
        self.file_format = file_format
        self.primers = self.parse_primers()
        self.coverage = coverage
        self._backend = _backend or _lib
        self.device = device

    def parse_primers(self):
        """extract_PCR_product_V1.py:141-167"""
        return parse_primers(self.primers_file, self.file_format)

    # -- device part ----------------------------------------------------------------------------------------
    def _hits(self, lines):
        """all occurrences of all expansions of every forward primer and of the reverse complement of every reverse
        primer in every sequence line -> {(pattern index, line index): [positions ascending]}"""
        n = len(lines)
        width = max((len(s) for s in lines), default=0)
        pats, lens_p = [], []
        for f, r in self.primers.values():
            for p, masks in ((f, allow_of(f)), (r, allow_rc_of(r))):
                if not 1 <= len(p) <= 32:
                    raise SystemExit("Error: primers of 1..32 bases are supported (%s)" % p)
                pats.append(masks)
                lens_p.append(len(p))
        out = {}
        if n == 0 or width == 0 or not pats:
            return out
        table = np.zeros(256, np.uint8)
        for ch, bit in _BASE_BIT.items():      # upper-case A, C, G, T only: the reference's search is plain text
            table[ord(ch)] = bit
        codes = np.zeros((n, width), np.uint8)
        lens = np.zeros(n, np.int32)
        for i, s in enumerate(lines):
            b = np.frombuffer(s.encode("latin-1", "replace"), np.uint8)
            codes[i, :len(b)] = table[b]
            lens[i] = len(b)
        ctx = self._backend.Context.shared(self.device) if hasattr(self._backend.Context, "shared") else \
            self._backend.Context(self.device)
        msa = self._backend.Msa(ctx, pack4(codes), n, width, lens=lens)
        try:
            hp, hr, hx = msa.pattern_hits(np.array(pats, np.uint32), np.array(lens_p, np.int32))
        finally:
            msa.close()
        for p, r, x in zip(hp.tolist(), hr.tolist(), hx.tolist()):
            out.setdefault((p, r), []).append(x)
        return out

    # -- the reference's choice among the hits ----------------------------------------------------------------
    @staticmethod
    def _product(line, f, r, f_pos, r_pos):
        """extract_PCR_product_V1.py:193-211 for one sequence line, given the positions where expansions of F / reverse
        complements of expansions of R occur in it"""
        if not f_pos or not r_pos:
            return ""
        kf, kr = len(f), len(r)
        f_rank = {e: i for i, e in enumerate(expansion_order(f))}
        r_rank = {RC(e): i for i, e in enumerate(expansion_order(r))}
        by_exp = {}
        for x in f_pos:
            by_exp.setdefault(line[x:x + kf], []).append(x)
        for e in sorted(by_exp, key=lambda s: f_rank[s]):
            xs = by_exp[e]
            x1 = xs[0]
            x2 = next((x for x in xs[1:] if x >= x1 + kf), None)       # str.split: non-overlapping occurrences
            end = len(line) if x2 is None else x2
            best = None
            for p in r_pos:
                if p >= x1 and p + kr <= end:
                    t = line[p:p + kr]
                    key = (r_rank[t], p)                                # first expansion of R in order, then leftmost
                    if best is None or key < best[0]:
                        best = (key, p, t)
            if best is not None:
                _, p, t = best
                return line[x1:p].strip() + t
        return ""

    def run(self):
        if not self.output_file.exists():
            os.makedirs(self.output_file, exist_ok=True)
        keys, lines = [], []
        with open(self.ref_file, "r") as fh:                           # every non-header LINE is searched on its own
            key = None
            for raw in fh:
                if raw.startswith(">"):
                    key = raw.strip()
                else:
                    keys.append(key)
                    lines.append(raw)
        hits = self._hits(lines)
        product_ids, non_product_ids = set(), set()
        for pi, (name, (f, r)) in enumerate(self.primers.items()):
            product_dict, non_targets = {}, {}
            for li, (key, line) in enumerate(zip(keys, lines)):
                value = self._product(line, f, r, hits.get((2 * pi, li)), hits.get((2 * pi + 1, li)))
                if value:
                    product_dict[key] = value
                else:
                    non_targets[key] = line.strip()
            with open(self.coverage, "a+") as c:
                c.write("Number of Product/non_Product, primer-F and primer-R: {}\t{}\t{}\t{}\t{}\n".format(
                    name, len(product_dict), len(non_targets), f, r))
            with open(Path(self.output_file).joinpath(name).with_suffix(".PCR.product.fa"), "w") as p:
                for k in product_dict:
                    product_ids.add(k)
                    p.write(k + "\n" + product_dict[k] + "\n")
            with open(Path(self.output_file).joinpath(name).with_suffix(".non_PCR.product.fa"), "w") as p:
                for k in non_targets:
                    non_product_ids.add(k)
                    p.write(k + "\n" + non_targets[k] + "\n")
        with open(self.ref_file, encoding="utf-8") as f:
            seq_number = int(f.read().count("\n") / 2)
        with open(self.coverage, "a+") as c:
            c.write("Total number of sequences:\t{}\nCoveraged number of sequence:\t{}\nRate of coverage:\t>= {}\n".format(
                seq_number, len(product_ids), round(float(len(product_ids)) / seq_number, 2)))


def allow_rc_of(primer: str):
    """allowed-base masks of the reverse complements of a primer's expansions"""
    comp = {"A": "T", "C": "G", "G": "C", "T": "A"}
    k = len(primer)
    allow = [0, 0, 0, 0]
    for i, ch in enumerate(primer):
        for base in DEGENERATE_BASE.get(ch, [ch]):
            if base in comp:
                allow["ACGT".index(comp[base])] |= 1 << (k - 1 - i)
    return allow


def main(argv=None, _backend=None):
    e1 = time.time()
    options = argsParse(argv)
    app = Product(primer_file=options.input, output_file=options.out, ref_file=options.ref, file_format=options.format,
                  coverage=options.stast, nproc=options.process, device=options.device, _backend=_backend)
    app.run()
    e2 = time.time()
    print("INFO {} Total times: {}".format(time.strftime("%Y-%m-%d %H:%M:%S", time.localtime(time.time())),
                                           round(float(e2 - e1), 2)))


if __name__ == "__main__":
    main()
