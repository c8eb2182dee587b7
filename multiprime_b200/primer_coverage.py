"""In-silico PCR of a primer set against unaligned targets, with mismatches, on both strands: which targets does each
pair of the set amplify, and how many does the set amplify as a whole.  It checks a designed set under the same mismatch
rule the core designed it with (-v, -c), against the raw sequences or against a background database (another -r).

Semantics
  Targets   FASTA records may span several lines; the lines of a record are joined.  Case is folded and U is read as T;
            IUPAC letters keep their base set; '-' and '.' are removed (alignment gaps are not bases); every other
            character becomes N.  A record is named by the first word of its header.
  Cell      A target cell matches a primer position only when the cell holds exactly one base and the primer allows that
            base (mpb_pattern_hits' rule): IUPAC and N cells in a target are always mismatches.
  Site      Primer P of length L binds at position x when the site lies inside one record, at most v positions mismatch
            and no mismatch falls on a strict position.  Strict positions come from core.strict_masks(-c, L) as
            mis_primer_check applies them: the forward primer F uses fmask over its own positions, the reverse primer R
            uses rmask over the positions of RC(R) (the window orientation of the core).  So a window primer the core
            scored gets the same per-sequence verdict here.
  Patterns  Four per pair, all searched on the stored strand: F (fmask), RC(R) (rmask), R (rmask bit-reversed over L_R),
            RC(F) (fmask bit-reversed over L_F).
  Amplicon  + strand: an F site at x and an RC(R) site at y >= x + L_F with product length y + L_R - x in [lo, hi];
            - strand: an R site at x and an RC(F) site at y >= x + L_R with length y + L_F - x in [lo, hi].
            A target is amplified by a pair when it has at least one amplicon.  The reported amplicon has the fewest
            total mismatches, then is the shortest, then + before -, then has the smallest x.
  Limits    primers of 1..32 bases, 0 <= v <= 15 and v smaller than every primer's length, 0 < lo <= hi.

Layout: all records are concatenated into one stream with L_max gap cells between records, and the stream is cut into rows
of S + L_max - 1 columns that start every S columns, so any mix of short records and multi-megabase genomes uploads as a
dense column view.  A site is kept only in the row whose first S columns hold its start, and only when it lies inside one
record.  The search is mpb_pattern_sites; pairing sites into amplicons is sort-based numpy.  Under torchrun every rank
searches a contiguous block of rows and rank 0 gathers the sites, pairs them and writes the files.

Outputs: <out>.amplicons.tsv (one row per pair and amplified target, pair order then target order; Start / End 0-based,
half-open, on the record as given) and <out>.coverage.tsv (one row per pair and an ALL row for the union over the set)."""
from __future__ import annotations

import sys
import time
from optparse import SUPPRESS_HELP, OptionParser

import numpy as np

from . import _lib
from .core import pack4, strict_masks
from .iupac import CHAR_CODE
from .pcr_product import allow_of, allow_rc_of, parse_primers

S = 4096              # stream columns per row: rows are S + L_max - 1 wide, so the row overlap costs < 1 %
MAX_V = 15            # the saturating counter of the column scan
MAX_PRIMER = 32       # bits of a pattern mask
_DROP = 255

_CODE = np.full(256, 15, np.uint8)                 # every other character -> N
for _ch, _c in CHAR_CODE.items():
    if _ch != "-":
        _CODE[ord(_ch)] = _CODE[ord(_ch.lower())] = _c
_CODE[ord("U")] = _CODE[ord("u")] = CHAR_CODE["T"]
for _ch in "-.\n\r":
    _CODE[ord(_ch)] = _DROP

AMPLICON_HEADER = "#Pair\tTarget\tStrand\tStart\tEnd\tLength\tF_mismatches\tR_mismatches\n"
COVERAGE_HEADER = "#Pair\tPrimer_F\tPrimer_R\tAmplified\tPerfect\tTotal\tCoverage\n"


class Targets:
    """records of a FASTA as one array of 4-bit base sets: record r is codes[off[r]:off[r] + lens[r]]"""

    def __init__(self, names, codes, lens):
        self.names = names
        self.codes = codes
        self.lens = np.asarray(lens, np.int64)
        self.off = np.concatenate([[0], np.cumsum(self.lens)]).astype(np.int64)


def read_targets(path: str) -> Targets:
    data = np.fromfile(path, np.uint8)
    nl = np.flatnonzero(data == 10)
    line_starts = np.concatenate([[0], nl + 1])
    line_starts = line_starts[line_starts < len(data)]
    hs = line_starts[data[line_starts] == ord(">")]                 # header line starts
    he = nl[np.searchsorted(nl, hs)] if len(nl) else np.zeros(0, np.int64)
    if len(he) < len(hs):                                           # a last header line without a newline
        he = np.concatenate([he, np.full(len(hs) - len(he), len(data))])
    he = np.minimum(he, len(data))
    delta = np.zeros(len(data) + 1, np.int8)
    delta[hs] += 1
    delta[he] -= 1
    keep = np.cumsum(delta[:-1], dtype=np.int8) == 0
    mapped = _CODE[data]
    keep &= mapped != _DROP
    if not len(hs):
        raise SystemExit("Error: %s holds no FASTA record" % path)
    if keep[:hs[0]].any():
        raise SystemExit("Error: %s has sequence text before its first '>' header" % path)
    lens = np.add.reduceat(keep.view(np.uint8), hs, dtype=np.int64)
    names = []
    for a, b in zip(hs.tolist(), he.tolist()):
        words = data[a + 1:b].tobytes().decode("latin-1").split()
        names.append(words[0] if words else "")
    return Targets(names, mapped[keep], lens)


class Panel:
    """the four search patterns of every pair, in the order F, RC(R), R, RC(F)"""

    def __init__(self, pairs: dict, coordinate: str):
        self.names = list(pairs)
        self.primers = [(f.strip().upper(), r.strip().upper()) for f, r in pairs.values()]
        allow, plen, strict = [], [], []
        for f, r in self.primers:
            for p in (f, r):
                if not 1 <= len(p) <= MAX_PRIMER:
                    raise SystemExit("Error: primers of 1..%d bases are supported (%r has %d)" % (MAX_PRIMER, p, len(p)))
            fmask, rmask = strict_masks(coordinate, len(f))[0], strict_masks(coordinate, len(r))[1]
            allow += [allow_of(f), allow_rc_of(r), allow_of(r), allow_rc_of(f)]
            plen += [len(f), len(r), len(r), len(f)]
            strict += [fmask, rmask, _reverse(rmask, len(r)), _reverse(fmask, len(f))]
        self.allow = np.array(allow, np.uint32).reshape(-1, 4)
        self.plen = np.array(plen, np.int32)
        self.strict = np.array(strict, np.uint32)
        self.lmax = int(self.plen.max()) if len(plen) else 1


def _reverse(mask: int, n: int) -> int:
    return sum(1 << (n - 1 - i) for i in range(n) if (mask >> i) & 1)


def layout(targets: Targets, lmax: int):
    """rows of the stream (records separated by lmax gap cells), nibble-packed -> (packed [n_rows, row_bytes], width,
    stream offset of every record)"""
    starts = np.concatenate([[0], np.cumsum(targets.lens + lmax)]).astype(np.int64)
    n_rows = max(1, -(-int(starts[-1]) // S))
    width = S + lmax - 1
    row_bytes = (width + 1) // 2
    stream = np.zeros(n_rows * S + 2 * lmax + 2, np.uint8)
    for a, o, n in zip(starts[:-1].tolist(), targets.off[:-1].tolist(), targets.lens.tolist()):
        stream[a:a + n] = targets.codes[o:o + n]
    packed = pack4(stream[None, :])[0]
    rows = np.lib.stride_tricks.as_strided(packed, (n_rows, row_bytes), (S // 2, 1))
    return np.ascontiguousarray(rows), width, starts[:-1]


def stream_sites(hp, hr, hx, hm, plen, starts, lens):
    """row sites -> (pattern, record, position in the record, mismatches) of the sites that start in the first S columns
    of their row and lie inside one record"""
    g = hr.astype(np.int64) * S + hx
    rec = np.searchsorted(starts, g, side="right") - 1
    keep = (hx < S) & (rec >= 0)
    rec = np.maximum(rec, 0)
    keep &= g + plen[hp] <= starts[rec] + lens[rec]
    return hp[keep], rec[keep], (g - starts[rec])[keep], hm[keep]


def find_sites(targets: Targets, panel: Panel, v: int, device=0, comm=None, backend=None, stream=None):
    """(pattern, record, position, mismatches) int64 arrays of every site, on rank 0 (None on the other ranks)"""
    backend = backend or _lib
    rank, world = (comm.rank, comm.world) if comm is not None else (0, 1)
    rows, width, starts = layout(targets, panel.lmax)
    lo, hi = rank * len(rows) // world, (rank + 1) * len(rows) // world
    quad = np.zeros((0, 4), np.int32)
    if hi > lo:
        ctx = backend.Context.shared(device, stream)
        msa = backend.Msa(ctx, rows[lo:hi], hi - lo, width, row_bytes=rows.shape[1])
        try:
            hp, hr, hx, hm = msa.pattern_sites(panel.allow, panel.plen, panel.strict, v, max_hits=1 << 22)
        finally:
            msa.close()
        quad = np.stack([hp, np.asarray(hr) + lo, hx, hm], 1).astype(np.int32)
    if comm is not None and world > 1:
        flat, _ = comm.allgather_concat(quad.reshape(-1))
        quad = flat.reshape(-1, 4)
        if rank != 0:
            return None
    quad = quad.astype(np.int64)
    return stream_sites(quad[:, 0], quad[:, 1], quad[:, 2], quad[:, 3], panel.plen.astype(np.int64), starts,
                        targets.lens)


def amplicons(sites, panel: Panel, lens, lo: int, hi: int, v: int):
    """best amplicon of every (pair, amplified target) -> list per pair of dict of int64 arrays (rec, strand, start, end,
    length, fmis, rmis), records ascending"""
    sp, srec, spos, smis = sites
    order = np.lexsort((spos, srec, sp))
    sp, srec, spos, smis = sp[order], srec[order], spos[order], smis[order]
    bounds = np.searchsorted(sp, np.arange(len(panel.plen) + 1))
    big = int(lens.max()) + 1 if len(lens) else 1

    def of(p):
        a, b = bounds[p], bounds[p + 1]
        return srec[a:b], spos[a:b], smis[a:b]

    out = []
    for q in range(len(panel.names)):
        lf, lr = int(panel.plen[4 * q]), int(panel.plen[4 * q + 1])
        cand = []
        for strand, (left, right, ll, rl) in enumerate(((4 * q, 4 * q + 1, lf, lr), (4 * q + 2, 4 * q + 3, lr, lf))):
            lrec, lx, lm = of(left)
            rrec, ry, rm = of(right)
            ylo = lx + max(ll, lo - rl)
            yhi = np.minimum(lx + hi - rl, big - 1)
            qlo, qhi = lrec * big + ylo, lrec * big + yhi
            found = np.zeros(len(lx), bool)
            y = np.zeros(len(lx), np.int64)
            mr = np.zeros(len(lx), np.int64)
            for m in range(v + 1):                     # the fewest right-site mismatches first, then the nearest site
                keys = np.sort(rrec[rm == m] * big + ry[rm == m])
                if not len(keys):
                    continue
                i = np.searchsorted(keys, qlo)
                k = keys[np.minimum(i, len(keys) - 1)]
                hit = ~found & (i < len(keys)) & (k <= qhi) & (ylo <= yhi)
                y[hit] = k[hit] - lrec[hit] * big
                mr[hit] = m
                found |= hit
            f = found
            length = y[f] + rl - lx[f]
            fm, rmm = (lm[f], mr[f]) if strand == 0 else (mr[f], lm[f])
            cand.append((lrec[f], lm[f] + mr[f], length, np.full(int(f.sum()), strand, np.int64), lx[f], fm, rmm))
        rec, tot, length, st, x, fm, rmm = (np.concatenate(c) for c in zip(*cand))
        o = np.lexsort((x, st, length, tot, rec))
        rec, uniq = np.unique(rec[o], return_index=True)
        pick = o[uniq]
        out.append(dict(rec=rec, strand=st[pick], start=x[pick], end=x[pick] + length[pick], length=length[pick],
                        fmis=fm[pick], rmis=rmm[pick]))
    return out


def write_outputs(out: str, panel: Panel, targets: Targets, best):
    n = len(targets.names)
    amplified = np.zeros(n, bool)
    perfect = np.zeros(n, bool)
    with open(out + ".amplicons.tsv", "w") as fa, open(out + ".coverage.tsv", "w") as fc:
        fa.write(AMPLICON_HEADER)
        fc.write(COVERAGE_HEADER)
        for name, (f, r), b in zip(panel.names, panel.primers, best):
            fa.writelines("%s\t%s\t%s\t%d\t%d\t%d\t%d\t%d\n" % (name, targets.names[rec], "+-"[st], s, e, ln, fm, rm)
                          for rec, st, s, e, ln, fm, rm in zip(*(b[k].tolist() for k in
                                                                  ("rec", "strand", "start", "end", "length", "fmis",
                                                                   "rmis"))))
            perf = b["rec"][(b["fmis"] + b["rmis"]) == 0]
            amplified[b["rec"]] = True
            perfect[perf] = True
            fc.write("%s\t%s\t%s\t%d\t%d\t%d\t%s\n" % (name, f, r, len(b["rec"]), len(perf), n,
                                                       round(len(b["rec"]) / n, 4)))
        fc.write("ALL\t-\t-\t%d\t%d\t%d\t%s\n" % (amplified.sum(), perfect.sum(), n, round(int(amplified.sum()) / n, 4)))


def check_limits(panel: Panel, v: int, lo: int, hi: int):
    if not 0 <= v <= MAX_V:
        raise SystemExit("Error: -v must be in 0..%d (got %d)" % (MAX_V, v))
    if len(panel.plen) and v >= int(panel.plen.min()):
        raise SystemExit("Error: -v %d is not smaller than the shortest primer (%d bases): every position would bind"
                         % (v, int(panel.plen.min())))
    if not 0 < lo <= hi:
        raise SystemExit("Error: -s needs 0 < lo <= hi (got %d,%d)" % (lo, hi))


def run(ref: str, pairs: dict, out: str, v: int = 1, coordinate: str = "1,2,-1", size=(50, 2000), device=0, comm=None,
        _backend=None):
    lo, hi = size
    panel = Panel(pairs, coordinate)
    if not panel.names:
        raise SystemExit("Error: no primer pair in the primer file")
    check_limits(panel, v, lo, hi)
    targets = read_targets(ref)
    sites = find_sites(targets, panel, v, device, comm, _backend)
    if sites is None:
        return None
    best = amplicons(sites, panel, targets.lens, lo, hi, v)
    write_outputs(out, panel, targets, best)
    return best


def argsParse(argv=None):
    parser = OptionParser('Usage: %prog -r [targets.fa] -i [primers] -f [format] -o [out_prefix]')
    parser.add_option('-r', '--ref', dest='ref', help='targets: FASTA of unaligned sequences (or a background database).')
    parser.add_option('-i', '--input', dest='input',
                      help='Primer file. One of: final_maxprimers_set.xls, primer.fa, primer_F,primer_R.')
    parser.add_option('-f', '--format', dest='format', help='Format of primer file: xls or fa or seq.')
    parser.add_option('-o', '--out', dest='out', default="primer_coverage",
                      help='Output prefix: <out>.amplicons.tsv and <out>.coverage.tsv. default: primer_coverage.')
    parser.add_option('-v', '--variation', dest='variation', default=1, type="int",
                      help='Max mismatch number of a primer site. Default: 1.')
    parser.add_option('-c', '--coordinate', dest='coordinate', default="1,2,-1",
                      help='Primer positions where a mismatch disqualifies a site (>0: from the 5\' end, <0: from the 3\' '
                           'end). Default: 1,2,-1.')
    parser.add_option('-s', '--size', dest='size', default="50,2000", help='lo,hi of the product length. Default: 50,2000.')
    parser.add_option('--device', dest='device', default=0, type="int", help=SUPPRESS_HELP)
    args = sys.argv[1:] if argv is None else argv
    (options, rest) = parser.parse_args(args)
    for value, msg in ((options.ref, "Input (targets) file must be specified !!!"),
                       (options.input, "Primer file or sequence must be specified !!!"),
                       (options.format, "Primer file format must be specified !!!")):
        if value is None:
            parser.print_help(sys.stderr)
            raise SystemExit("Error: " + msg)
    if options.format not in ("xls", "fa", "seq"):
        raise SystemExit("Error: -f must be xls, fa or seq (got %s)" % options.format)
    try:
        options.size = tuple(int(x) for x in options.size.split(","))
        assert len(options.size) == 2
        strict_masks(options.coordinate, 32)
    except (ValueError, AssertionError):
        raise SystemExit("Error: -s takes lo,hi and -c a comma-separated list of integers")
    return options


def main(argv=None, _backend=None):
    from .findimer import shard_setup
    e1 = time.time()
    options = argsParse(argv)
    extra, rank = shard_setup(options.device)
    run(options.ref, parse_primers(options.input, options.format), options.out, options.variation, options.coordinate,
        options.size, _backend=_backend, **extra)
    if "comm" in extra:
        import torch.distributed as dist
        dist.destroy_process_group()
    e2 = time.time()
    if rank == 0:
        print("INFO {} Total times: {}".format(time.strftime("%Y-%m-%d %H:%M:%S", time.localtime(time.time())),
                                               round(float(e2 - e1), 2)))


if __name__ == "__main__":
    main()
