"""In-silico PCR over every primer combination of a multiplex set: what else does the set amplify when all its primers
share one tube?  primer_coverage checks each pair's own products; this tool joins every primer's left sites with every
primer's right sites, so it also finds the products of primers of different pairs and of one primer binding on both
strands, on the targets or on a background database (another -r).

Semantics
  Targets, cells, sites, strict masks, limits, stream layout and primer files are primer_coverage's (read_targets,
  Panel, check_limits, layout, parse_primers).
  Primers   The set's primers in order F_0, R_0, F_1, R_1, ... (primer 2q = F_q, 2q + 1 = R_q), named <pair>:F and
            <pair>:R.  Each keeps its strict positions of primer_coverage: F uses fmask; R uses rmask read as positions
            of R itself.
  Sites     Primer i has a left site at x when i itself binds there on the stored strand, and a right site at y when
            RC(i) binds there: Panel's patterns 4q (F_q) and 4q+2 (R_q) are left sites, 4q+1 (R_q) and 4q+3 (F_q) right
            sites.
  Product   (i, j): a left site of i at x and a right site of j at y in one record, with y >= x + L_i and a length
            y + L_j - x in [lo, hi].  Any i and j form products, i = j included.  (F_q, R_q) is primer_coverage's +
            amplicon and (R_q, F_q) its - amplicon.
  Class     of a combination (i, j), decided by sequence: intended when (seq i, seq j) is (F_q, R_q) or (R_q, F_q) of
            some pair q; otherwise self when seq i = seq j; otherwise cross.  So a primer listed in two pairs is not
            reported as its own cross product.
  Group     (target, i, j) with at least one product.  It carries its number of products and its best product: the
            fewest total mismatches, then the shortest, then the smallest start.

The search and the join run on the device (mpb_pattern_products): the sites never leave HBM, only the per-combination
summaries and the listed groups come back.  Under torchrun the ranks take contiguous whole records, split near an even
share of stream columns; a row that holds columns of two ranks' records is searched by both and each keeps the sites of
its own records, so the per-rank summaries add exactly.  Rank 0 gathers them and the ranks' listed rows in rank order.

Outputs
  <out>.specificity.tsv  one row per combination with at least one product, in (i, j) order: products, targets with a
                         group, targets whose best product has no mismatch, number of records; then an UNINTENDED row,
                         the union over every combination that is not intended.  Always exact.
  <out>.products.tsv     one row per group of a combination that is not intended, in order of target (file order), i,
                         j; Start / End 0-based and half-open on the record as given.  Only the first --max-rows rows
                         are written; stderr says so when that cuts the list.  Intended products are primer_coverage's
                         to list."""
from __future__ import annotations

import sys
import time
from optparse import SUPPRESS_HELP, OptionParser

import numpy as np

from . import _lib
from . import primer_coverage as pc
from .pcr_product import parse_primers

MAX_ROWS = 1_000_000
SPECIFICITY_HEADER = "#Left\tRight\tClass\tProducts\tTargets\tPerfect_targets\tTotal\n"
PRODUCTS_HEADER = "#Left\tRight\tClass\tTarget\tStart\tEnd\tLength\tLeft_mismatches\tRight_mismatches\tProducts\n"
CLASSES = ("intended", "self", "cross")


class Primers:
    """the primers of a Panel (2q = F_q, 2q + 1 = R_q), the primer and side of each of its patterns, and the class of
    every combination"""

    def __init__(self, panel: pc.Panel):
        self.names = [n + s for n in panel.names for s in (":F", ":R")]
        self.seqs = [p for fr in panel.primers for p in fr]
        q = np.arange(len(panel.plen)) // 4
        self.pat_primer = (2 * q + np.array([0, 1, 1, 0], np.int32)[np.arange(len(panel.plen)) % 4]).astype(np.int32)
        self.pat_side = np.tile(np.array([0, 1, 0, 1], np.int32), len(panel.names))
        intended = {fr for f, r in panel.primers for fr in ((f, r), (r, f))}
        n = len(self.seqs)
        self.klass = np.zeros((n, n), np.int8)
        for i, a in enumerate(self.seqs):
            for j, b in enumerate(self.seqs):
                self.klass[i, j] = 0 if (a, b) in intended else 1 if a == b else 2
        self.listed = (self.klass != 0).astype(np.uint8)


def shard_records(targets: pc.Targets, lmax: int, world: int):
    """record bounds [world + 1] of the ranks: contiguous whole records near an even share of stream columns"""
    starts = np.concatenate([[0], np.cumsum(targets.lens + lmax)]).astype(np.int64)
    cut = np.searchsorted(starts[:-1], np.arange(world + 1) * (int(starts[-1]) / world), side="left")
    cut[0], cut[-1] = 0, len(targets.lens)
    return np.maximum.accumulate(cut)


def find_groups(targets: pc.Targets, panel: pc.Panel, v: int, lo: int, hi: int, listed, max_rows: int = MAX_ROWS,
                device=0, comm=None, backend=None, stream=None, chunk: int = 0):
    """products of every combination -> on rank 0 dict(comb int64[P, P, 3] (products, targets, perfect targets),
    union int64[2], rows int64[n, 8] (record, i, j, start, length, left mismatches, right mismatches, products) of the
    first max_rows groups of the combinations flagged in listed[P, P], n_listed, stats int64[4]); None on other ranks"""
    backend = backend or _lib
    primers = Primers(panel)
    n_primer = len(primers.seqs)
    rank, world = (comm.rank, comm.world) if comm is not None else (0, 1)
    rows, width, starts = pc.layout(targets, panel.lmax)
    bounds = shard_records(targets, panel.lmax, world)
    a, b = int(bounds[rank]), int(bounds[rank + 1])
    comb = np.zeros((n_primer, n_primer, 3), np.int64)
    sums = np.zeros(7, np.int64)                       # union[2], n_listed, stats[4]
    listed_rows = np.zeros((0, 8), np.int64)
    if b > a:
        end = int(starts[b - 1] + targets.lens[b - 1])
        row0 = int(starts[a]) // pc.S
        row1 = max(row0 + 1, -(-end // pc.S))
        ctx = backend.Context.shared(device, stream)
        msa = backend.Msa(ctx, rows[row0:row1], row1 - row0, width, row_bytes=rows.shape[1])
        try:
            res = msa.pattern_products(panel.allow, panel.plen, panel.strict, v, primers.pat_primer, primers.pat_side,
                                       n_primer, pc.S, starts[a:b] - row0 * pc.S, targets.lens[a:b], lo, hi, listed,
                                       max_rows, chunk)
        finally:
            msa.close()
        comb = res["comb"]
        sums = np.concatenate([res["union"], [res["n_listed"]], res["stats"]]).astype(np.int64)
        listed_rows = np.array(res["rows"], np.int64).reshape(-1, 8)
        listed_rows[:, 0] += a
    if comm is not None and world > 1:
        total = comm.allreduce_sum(np.concatenate([comb.reshape(-1), sums]))
        comb, sums = total[:comb.size].reshape(comb.shape), total[comb.size:]
        flat, _ = comm.allgather_concat(listed_rows.reshape(-1))
        listed_rows = flat.reshape(-1, 8)[:max_rows]
        if rank != 0:
            return None
    return dict(comb=comb, union=sums[:2], rows=listed_rows, n_listed=int(sums[2]), stats=sums[3:])


def write_outputs(out: str, primers: Primers, targets: pc.Targets, res, max_rows: int):
    n = len(targets.names)
    comb, names = res["comb"], primers.names
    with open(out + ".specificity.tsv", "w") as fs:
        fs.write(SPECIFICITY_HEADER)
        for i, j in zip(*np.nonzero(comb[:, :, 1])):
            fs.write("%s\t%s\t%s\t%d\t%d\t%d\t%d\n" % (names[i], names[j], CLASSES[primers.klass[i, j]], comb[i, j, 0],
                                                       comb[i, j, 1], comb[i, j, 2], n))
        fs.write("UNINTENDED\t-\t-\t%d\t%d\t%d\t%d\n" % (int(comb[:, :, 0][primers.klass != 0].sum()),
                                                         res["union"][0], res["union"][1], n))
    with open(out + ".products.tsv", "w") as fp:
        fp.write(PRODUCTS_HEADER)
        fp.writelines("%s\t%s\t%s\t%s\t%d\t%d\t%d\t%d\t%d\t%d\n" % (names[i], names[j], CLASSES[primers.klass[i, j]],
                                                                     targets.names[rec], s, s + ln, ln, lm, rm, k)
                      for rec, i, j, s, ln, lm, rm, k in res["rows"].tolist())
    if res["n_listed"] > len(res["rows"]):
        sys.stderr.write("Warning: --max-rows %d: %s.products.tsv lists %d of %d rows\n"
                         % (max_rows, out, len(res["rows"]), res["n_listed"]))


def run(ref: str, pairs: dict, out: str, v: int = 1, coordinate: str = "1,2,-1", size=(50, 2000), max_rows=MAX_ROWS,
        device=0, comm=None, _backend=None, _chunk: int = 0):
    lo, hi = size
    panel = pc.Panel(pairs, coordinate)
    if not panel.names:
        raise SystemExit("Error: no primer pair in the primer file")
    pc.check_limits(panel, v, lo, hi)
    if max_rows < 0:
        raise SystemExit("Error: --max-rows must be >= 0 (got %d)" % max_rows)
    targets = pc.read_targets(ref)
    primers = Primers(panel)
    try:
        res = find_groups(targets, panel, v, lo, hi, primers.listed, max_rows, device, comm, _backend, chunk=_chunk)
    except _lib.MpbError as exc:
        raise SystemExit("Error: %s" % exc)
    if res is None:
        return None
    write_outputs(out, primers, targets, res, max_rows)
    return res


def add_options(parser: OptionParser, out_default: str = "primer_specificity",
                out_help: str = "<out>.specificity.tsv and <out>.products.tsv"):
    """the flags -r -i -f -o -v -c -s of this tool; primer_pools takes them too"""
    parser.add_option('-r', '--ref', dest='ref', help='targets: FASTA of unaligned sequences (or a background database).')
    parser.add_option('-i', '--input', dest='input',
                      help='Primer file. One of: final_maxprimers_set.xls, primer.fa, primer_F,primer_R.')
    parser.add_option('-f', '--format', dest='format', help='Format of primer file: xls or fa or seq.')
    parser.add_option('-o', '--out', dest='out', default=out_default,
                      help='Output prefix: %s. default: %s.' % (out_help, out_default))
    parser.add_option('-v', '--variation', dest='variation', default=1, type="int",
                      help='Max mismatch number of a primer site. Default: 1.')
    parser.add_option('-c', '--coordinate', dest='coordinate', default="1,2,-1",
                      help='Primer positions where a mismatch disqualifies a site (>0: from the 5\' end, <0: from the 3\' '
                           'end). Default: 1,2,-1.')
    parser.add_option('-s', '--size', dest='size', default="50,2000", help='lo,hi of the product length. Default: 50,2000.')


def check_options(parser: OptionParser, options):
    """the checks of the flags of add_options (and of --max-rows when the parser has it); options.size -> (lo, hi)"""
    for value, msg in ((options.ref, "Input (targets) file must be specified !!!"),
                       (options.input, "Primer file or sequence must be specified !!!"),
                       (options.format, "Primer file format must be specified !!!")):
        if value is None:
            parser.print_help(sys.stderr)
            raise SystemExit("Error: " + msg)
    if options.format not in ("xls", "fa", "seq"):
        raise SystemExit("Error: -f must be xls, fa or seq (got %s)" % options.format)
    if getattr(options, "max_rows", 0) < 0:
        raise SystemExit("Error: --max-rows must be >= 0 (got %d)" % options.max_rows)
    try:
        options.size = tuple(int(x) for x in options.size.split(","))
        assert len(options.size) == 2
        pc.strict_masks(options.coordinate, 32)
    except (ValueError, AssertionError):
        raise SystemExit("Error: -s takes lo,hi and -c a comma-separated list of integers")
    return options


def argsParse(argv=None):
    parser = OptionParser('Usage: %prog -r [targets.fa] -i [primers] -f [format] -o [out_prefix]')
    add_options(parser)
    parser.add_option('--max-rows', dest='max_rows', default=MAX_ROWS, type="int",
                      help='Rows of <out>.products.tsv at most. Default: %d.' % MAX_ROWS)
    parser.add_option('--device', dest='device', default=0, type="int", help=SUPPRESS_HELP)
    args = sys.argv[1:] if argv is None else argv
    (options, rest) = parser.parse_args(args)
    return check_options(parser, options)


def main(argv=None, _backend=None):
    from .findimer import shard_setup
    e1 = time.time()
    options = argsParse(argv)
    extra, rank = shard_setup(options.device)
    run(options.ref, parse_primers(options.input, options.format), options.out, options.variation, options.coordinate,
        options.size, options.max_rows, _backend=_backend, **extra)
    if "comm" in extra:
        import torch.distributed as dist
        dist.destroy_process_group()
    e2 = time.time()
    if rank == 0:
        print("INFO {} Total times: {}".format(time.strftime("%Y-%m-%d %H:%M:%S", time.localtime(time.time())),
                                               round(float(e2 - e1), 2)))


if __name__ == "__main__":
    main()
