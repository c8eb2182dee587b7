"""Choose a multiplex primer set from a pool of candidate pairs by the targets it amplifies: the fewest pairs that
amplify the most targets, with no primer dimer between two chosen pairs.  get_Maxprimerset takes the first pair of each
cluster that passes the dimer check; this tool scores every candidate by in-silico PCR under primer_coverage's mismatch
rule and picks greedily.  With --keep it extends an existing panel: the kept pairs are taken first and the tool says
which candidates to add.

Semantics
  Candidates  -f xls, fa or seq: read with parse_primers.  -f sets: the one-line-per-cluster file of get_multiPrime
              (get_Maxprimerset's input): each line is split on tabs with empty fields dropped; field 0 is the cluster,
              then pairs follow as groups of five fields (F, R, product info, target number, start:stop; an incomplete
              last group is ignored).  A pair is named <cluster>_<start>_F_<cluster>_<stop> with cluster =
              field0.split("/")[-1].split(".")[0], the name parse_primers gives it in an xls; a name already read is
              skipped.  Candidate index = file order; it breaks every tie.
  Kept        --keep FILE (--keep-format xls, fa or seq) names pairs taken before any candidate.  A candidate with the
              name of a kept pair is that kept pair.
  Coverage    A(c): the targets where pair c has an amplicon by primer_coverage's rule (both strands, strict masks,
              product length in [lo, hi], both sites inside one record).  P(c) <= A(c): the targets where one such
              amplicon has no mismatch on either site.  |A(c)| and |P(c)| are the Amplified and Perfect columns of
              primer_coverage's coverage.tsv for c.
  Conflicts   Pairs a != b conflict when a primer of a and a primer of b have different sequences and finDimer's rule
              reports them (the dimer grid over the distinct sequences of the candidates and kept pairs: ends of 5..18,
              both initiation terms, loss_table(-t)); primer_pools counts the same dimers.  Dimers inside one pair are
              not considered.
  Cross       --cross: when a pair t is taken (kept pairs included), an eligible candidate c becomes ineligible when a
              primer i of one of {c, t} and a primer j of the other have a product on a target record (primer_specificity's
              rule: a left site of i at x and a right site of j at y in one record, y >= x + L_i, y + L_j - x in [lo, hi])
              and (i, j) is of class cross over the taken pairs plus c: (seq i, seq j) is no taken pair's and not c's
              (F, R) or (R, F), and seq i != seq j.  The dimers of a take are applied first.  Kept pairs are not checked
              against each other.
  Background  --background FILE (read as the targets, same -v -c -s): a candidate with a product of any of its own
              (F, R), (R, F), (F, F), (R, R) on a background record is off-target from the start and never a step's
              choice; kept pairs are taken regardless.  With --cross the cross products are also searched there.
  Greedy      Step 0 takes the kept pairs in file order, without a dimer check among them.  Taking a pair adds A and P
              to covered / covered_perfect, and every candidate that conflicts with it becomes ineligible.  Then, for
              steps s = 1, 2, ...: stop when -k pairs have been selected at steps >= 1 (k > 0); stop when covered /
              total >= goal; stop when no eligible candidate has gain = |A(c) minus covered| > 0; otherwise take the
              eligible candidate with the largest (gain, |P(c) minus covered_perfect|), the smallest index on ties.
              The result depends on the inputs and the flags only (not on the GPU, the blocks, the ranks or the order
              of the launches).
  Limits      primer_coverage's limits on primers, -v and -s; at most 16 384 candidate plus kept pairs; -k >= 0;
              0 < --goal <= 1; a coverage matrix that fits in device memory (2 * pairs + 2 rows of
              ceil(targets / 128) * 4 32-bit words).  The CLI refuses these before any search.

The matrix is built on the device (mpb_pattern_cover): blocks of pairs, each one pattern search and one join restricted
to each pair's own two patterns, one bit per (pair, target) left in HBM.  Each greedy step is one mpb_cover_gains call
over the eligible candidates (a candidate whose gain reached 0 stays at 0 and is not listed again) and one
mpb_cover_take.  Under torchrun every rank builds the columns of its own records (primer_specificity's record shards),
the gains of every step are summed over the ranks, so every rank takes the same pair, the dimer bands are dealt as in
finDimer, and rank 0 writes.  With --cross the cover calls also keep their sites in a resident site list (one search per
block still), sealed once into stream order; each take is one mpb_sites_cross (8 bits per pair: which primer of each
side is the left one), and the class rule is applied here from the sequences.  --background builds a second list from
search-only calls, joined once by mpb_sites_own.  Under torchrun each rank keeps the sites of its own records of both
files and the bits are OR-reduced over the ranks.

Outputs
  <out>.selected.tsv    one row per taken pair in step order: Amplified / Perfect are |A| / |P|, New / New_perfect the
                        gains when it was taken, Covered / Covered_perfect cumulative, Coverage = round(Covered / Total,
                        4).
  <out>.candidates.tsv  every candidate in input order with its Status: kept, selected, dimer or cross (Step / By: the
                        first taken pair that excluded it), off-target (Step 0, By -) or open (still eligible at the
                        stop).
  <out>.selected.fa     the taken pairs as four-line FASTA (headers <name>:F and <name>:R), for primer_specificity and
                        primer_pools -f fa."""
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

MAX_PAIRS = 16384
SITE_BUDGET = 1 << 26          # expected sites of one mpb_pattern_cover call: about 1 GB of keys and sort buffers
MAX_SITES = 1 << 31            # mpb_pattern_cover's largest first capacity
SELECTED_HEADER = ("#Step\tPair\tPrimer_F\tPrimer_R\tAmplified\tPerfect\tNew\tNew_perfect\tCovered\tCovered_perfect\t"
                   "Total\tCoverage\n")
CANDIDATES_HEADER = "#Pair\tPrimer_F\tPrimer_R\tAmplified\tPerfect\tStatus\tStep\tBy\n"


def read_sets(path: str) -> dict:
    """{pair name: (F, R)} of a get_multiPrime sets file, first occurrence of a name kept"""
    res = {}
    with open(path) as fh:
        for line in fh:
            row = list(filter(None, line.strip().split("\t")))
            if not row:
                continue
            cluster = row[0].split("/")[-1].split(".")[0]
            col = 1
            while col <= len(row) - 5:
                start, stop = row[col + 4].split(":")[:2]
                res.setdefault("%s_%s_F_%s_%s" % (cluster, start, cluster, stop), (row[col], row[col + 1]))
                col += 5
    return res


def read_candidates(path: str, fmt: str) -> dict:
    return read_sets(path) if fmt == "sets" else parse_primers(path, fmt)


class Pool:
    """the matrix rows: the kept pairs, then the candidates that are not kept; cand_row[i] is candidate i's row"""

    def __init__(self, cands: dict, keep: dict, coordinate: str):
        self.names = list(keep) + [n for n in cands if n not in keep]
        pairs = dict(keep)
        pairs.update((n, fr) for n, fr in cands.items() if n not in keep)
        self.panel = pc.Panel({str(i): pairs[n] for i, n in enumerate(self.names)}, coordinate)
        row = {n: i for i, n in enumerate(self.names)}
        self.n_keep = len(keep)
        self.cand_names = list(cands)
        self.cand_row = np.array([row[n] for n in cands], np.int64)


def check_select(n_pairs: int, max_pairs: int, goal: float):
    if n_pairs > MAX_PAIRS:
        raise SystemExit("Error: %d candidate and kept pairs: at most %d are supported" % (n_pairs, MAX_PAIRS))
    if max_pairs < 0:
        raise SystemExit("Error: -k must be >= 0 (got %d)" % max_pairs)
    if not 0 < goal <= 1:
        raise SystemExit("Error: --goal must be in (0, 1] (got %s)" % goal)


def block_of(n_rec: int, n_pairs: int) -> int:
    """pairs per mpb_pattern_cover call: about SITE_BUDGET sites when each of a pair's four patterns binds once per
    target"""
    return max(1, min(n_pairs, SITE_BUDGET // max(1, 4 * n_rec)))


def search_blocks(targets: pc.Targets, panel: pc.Panel, v: int, lo: int, hi: int, ctx, comm, backend, block: int,
                  mat, keep: bool, total):
    """the pattern search of this rank's records in blocks of pairs, into mat (None: no matrix) and, with keep, into
    a SiteList that is sealed and returned (None when the rank has no record); total += the stats of the calls"""
    n_pairs = len(panel.names)
    rank, world = (comm.rank, comm.world) if comm is not None else (0, 1)
    bounds = ps.shard_records(targets, panel.lmax, world)
    a, b = int(bounds[rank]), int(bounds[rank + 1])
    if b <= a:
        return None
    rows, width, starts = pc.layout(targets, panel.lmax)
    end = int(starts[b - 1] + targets.lens[b - 1])
    row0 = int(starts[a]) // pc.S
    row1 = max(row0 + 1, -(-end // pc.S))
    rec_off, rec_len = starts[a:b] - row0 * pc.S, targets.lens[a:b]
    sites = backend.SiteList(ctx, panel.plen, (row1 - row0) * pc.S, rec_off, rec_len) if keep else None
    msa = None
    try:
        msa = backend.Msa(ctx, rows[row0:row1], row1 - row0, width, row_bytes=rows.shape[1])
        # the search's capacity: the budget block_of sized the block by, then the previous block's sites with room to
        # spare, so a block's search runs once (mpb_pattern_cover searches again when its capacity is too small)
        cap = min(SITE_BUDGET, 4 * (b - a) * block)
        for p0 in range(0, n_pairs, block):
            p1 = min(n_pairs, p0 + block)
            args = (panel.allow[4 * p0:4 * p1], panel.plen[4 * p0:4 * p1], panel.strict[4 * p0:4 * p1], v, pc.S,
                    rec_off, rec_len, lo, hi, mat, p0, cap)
            st = msa.pattern_cover_keep(*args, sites) if keep else msa.pattern_cover(*args)
            total += st
            cap = int(min(MAX_SITES, max(cap, st[0] + st[0] // 4 + 1024)))
        if keep:
            sites.seal()
    except BaseException:
        if sites is not None:
            sites.close()
        raise
    finally:
        if msa is not None:
            msa.close()
    return sites


def build_matrix(targets: pc.Targets, panel: pc.Panel, v: int, lo: int, hi: int, device, comm, backend, block: int,
                 stats=None, keep_sites: bool = False):
    """the CoverMatrix of this rank's records (all pairs) and the total stats of the calls -> (ctx, mat); with
    keep_sites -> (ctx, mat, the sealed SiteList of the same search, None when the rank has no record)"""
    n_pairs = len(panel.names)
    rank, world = (comm.rank, comm.world) if comm is not None else (0, 1)
    bounds = ps.shard_records(targets, panel.lmax, world)
    a, b = int(bounds[rank]), int(bounds[rank + 1])
    ctx = backend.Context.shared(device)
    try:
        mat = backend.CoverMatrix(ctx, n_pairs, b - a)
    except _lib.MpbError as exc:
        raise SystemExit("Error: the coverage matrix of %d pairs x %d targets needs %d bytes of device memory (%s)"
                         % (n_pairs, b - a, _lib.cover_bytes(n_pairs, b - a), exc))
    total = np.zeros(3, np.int64)
    try:
        sites = search_blocks(targets, panel, v, lo, hi, ctx, comm, backend, block, mat, keep_sites, total)
    except BaseException:
        mat.close()
        raise
    if stats is not None:
        stats += total
    return (ctx, mat, sites) if keep_sites else (ctx, mat)


def products_of(sites, lo: int, hi: int, comm, n_rows: int, pair=None, eligible=None):
    """the per-pair bytes of SiteList.cross (pair given) or SiteList.own over the lists of this rank (None: a rank
    without records), OR-ed over the lists and the ranks"""
    bits = np.zeros(n_rows, np.uint8)
    for s in sites:
        if s is not None:
            bits |= s.own(lo, hi) if pair is None else s.cross(lo, hi, pair, eligible)
    if comm is not None and comm.world > 1:
        flags = comm.allreduce_sum(np.unpackbits(bits).astype(np.int64))
        bits = np.packbits(flags > 0)
    return bits


def off_target(sites, pool: Pool, lo: int, hi: int, comm) -> list:
    """the candidate rows (kept rows aside) with a product of their own primers on the background"""
    bits = products_of(sites, lo, hi, comm, len(pool.names))
    return [int(r) for r in np.nonzero(bits)[0] if r >= pool.n_keep]


def crosses(sites, pool: Pool, lo: int, hi: int, comm):
    """row, eligible bool[rows] -> the eligible rows that form a cross product with `row` on the lists' records.  Rows
    must be passed in the order they are taken: the intended combinations are those of the pairs taken so far"""
    prim = pool.panel.primers
    intended = set()

    def of(row, eligible):
        f, r = prim[row]
        intended.update(((f, r), (r, f)))
        if not eligible.any():
            return []
        bits = products_of(sites, lo, hi, comm, len(pool.names), row, eligible)
        out = []
        for c in np.nonzero(bits)[0].tolist():
            fc, rc = prim[c]
            for bit in range(8):
                if not bits[c] >> bit & 1:
                    continue
                sc, st = prim[c][bit >> 1 & 1], prim[row][bit & 1]
                i, j = (st, sc) if bit < 4 else (sc, st)
                if i != j and (i, j) not in intended and (i, j) not in ((fc, rc), (rc, fc)):
                    out.append(c)
                    break
        return out
    return of


def conflicts(panel: pc.Panel, hits, distinct):
    """row -> the other rows it conflicts with, from the dimer grid's hits over the distinct sequences.  The mapping of
    primer_pools.conflict_matrices, kept sparse: its dense primer x primer matrix would be 32 768^2 cells at 16 384 pairs"""
    index = {s: k for k, s in enumerate(distinct)}
    seq_rows = [[] for _ in distinct]
    row_seqs = []
    for q, (f, r) in enumerate(panel.primers):
        mine = sorted({index[f], index[r]})
        row_seqs.append(mine)
        for s in mine:
            seq_rows[s].append(q)
    partners = [set() for _ in distinct]
    for i, j, _, _ in hits:
        if i != j:
            partners[i].add(j)
            partners[j].add(i)

    def of(q):
        out = set()
        for s in row_seqs[q]:
            for t in partners[s]:
                out.update(seq_rows[t])
        out.discard(q)
        return sorted(out)
    return of


def greedy(ctx, mat, pool: Pool, conflict_of, n_targets: int, max_pairs: int, goal: float, comm=None, cross_of=None,
           off=()):
    """-> (amp[n_rows, 2] = |A|, |P|; taken [(row, step, new, new_perfect)]; excluded {row: (step, by row or None,
    status)}; taken rows set).  off: candidate rows excluded from the start (off-target); cross_of(row, eligible
    bool[n_rows]): the eligible rows that taking `row` excludes as cross products (after its dimers)"""
    def gains(rows):
        g = ctx.cover_gains(mat, np.asarray(rows, np.int32))
        if comm is not None and comm.world > 1:
            g = comm.allreduce_sum(g.reshape(-1)).reshape(-1, 2)
        return g

    n_rows = len(pool.names)
    size = gains(np.arange(n_rows))
    taken, excluded, done = [], {r: (0, None, "off-target") for r in off}, set()
    covered = 0

    def take(row, step, g):
        nonlocal covered
        ctx.cover_take(mat, row)
        taken.append((row, step, int(g[0]), int(g[1])))
        done.add(row)
        covered += int(g[0])
        for c in conflict_of(row):
            if c >= pool.n_keep and c not in done and c not in excluded:
                excluded[c] = (step, row, "dimer")
        if cross_of is not None:
            eligible = np.zeros(n_rows, bool)
            eligible[pool.n_keep:] = True
            eligible[list(done) + list(excluded)] = False
            for c in cross_of(row, eligible):
                excluded[c] = (step, row, "cross")

    for row in range(pool.n_keep):
        take(row, 0, gains([row])[0])
    live = np.unique(pool.cand_row[pool.cand_row >= pool.n_keep])        # rows in index order
    step = 0
    while True:
        if max_pairs and step >= max_pairs:
            break
        if covered / n_targets >= goal:
            break
        live = np.array([r for r in live.tolist() if r not in excluded and r not in done], np.int64)
        if not len(live):
            break
        g = gains(live)
        key = g[:, 0] * (n_targets + 1) + g[:, 1]
        k = int(np.argmax(key))                  # the first maximum: the smallest index
        if g[k, 0] == 0:
            break
        step += 1
        take(int(live[k]), step, g[k])
        live = live[g[:, 0] > 0]                 # gains never grow: a zero stays zero
    return size, taken, excluded, done


def write_outputs(out: str, pool: Pool, size, taken, excluded, n_targets: int):
    names, prim = pool.names, pool.panel.primers
    step_of = {}
    with open(out + ".selected.tsv", "w") as fo, open(out + ".selected.fa", "w") as ff:
        fo.write(SELECTED_HEADER)
        cov = covp = 0
        for row, step, new, newp in taken:
            cov += new
            covp += newp
            step_of[row] = step
            fo.write("%d\t%s\t%s\t%s\t%d\t%d\t%d\t%d\t%d\t%d\t%d\t%s\n" % (
                step, names[row], prim[row][0], prim[row][1], size[row, 0], size[row, 1], new, newp, cov, covp,
                n_targets, round(cov / n_targets, 4)))
            ff.write(">%s:F\n%s\n>%s:R\n%s\n" % (names[row], prim[row][0], names[row], prim[row][1]))
    with open(out + ".candidates.tsv", "w") as fo:
        fo.write(CANDIDATES_HEADER)
        for name, row in zip(pool.cand_names, pool.cand_row.tolist()):
            if row < pool.n_keep:
                status, step, by = "kept", "0", "-"
            elif row in step_of:
                status, step, by = "selected", str(step_of[row]), "-"
            elif row in excluded:
                s, t, status = excluded[row]
                step, by = str(s), "-" if t is None else names[t]
            else:
                status, step, by = "open", "-", "-"
            fo.write("%s\t%s\t%s\t%d\t%d\t%s\t%s\t%s\n" % (name, prim[row][0], prim[row][1], size[row, 0], size[row, 1],
                                                          status, step, by))


def run(ref: str, cands: dict, out: str, v: int = 1, coordinate: str = "1,2,-1", size=(50, 2000), max_pairs: int = 0,
        goal: float = 1.0, threshold: float = 3.96, keep=None, cross: bool = False, background=None, device=0, comm=None,
        _backend=None, _block: int = 0, _times=None, _stats=None):
    """-> dict(taken [(row, step, new, new_perfect)], names, size int64[rows, 2], covered) on rank 0, None elsewhere.
    cross: exclude the cross products of each taken pair; background: FASTA whose products exclude candidates"""
    backend = _backend or _lib
    lo, hi = size
    keep = keep or {}
    pool = Pool(cands, keep, coordinate)
    panel = pool.panel
    if not cands:
        raise SystemExit("Error: no candidate pair in the primer file")
    pc.check_limits(panel, v, lo, hi)
    check_select(len(pool.names), max_pairs, goal)
    times = _times if _times is not None else {}
    t0 = time.perf_counter()
    targets = pc.read_targets(ref)
    bg = pc.read_targets(background) if background else None
    n_targets = len(targets.names)
    sites = []
    try:
        t1 = time.perf_counter()
        built = build_matrix(targets, panel, v, lo, hi, device, comm, backend,
                             _block or block_of(len(targets.names), len(pool.names)), _stats, keep_sites=cross)
        ctx, mat = built[:2]
        sites = list(built[2:])
        try:
            t2 = time.perf_counter()
            off = []
            if bg is not None:
                sites.append(search_blocks(bg, panel, v, lo, hi, ctx, comm, backend,
                                           _block or block_of(len(bg.names), len(pool.names)), None, True,
                                           np.zeros(3, np.int64)))
                off = off_target(sites[-1:], pool, lo, hi, comm)
            t3 = time.perf_counter()
            distinct = list(dict.fromkeys(s for fr in panel.primers for s in fr))
            hits, _, _ = grid_hits(ctx, backend, [sets_of(s) for s in distinct], threshold, comm)
            t4 = time.perf_counter()
            amp, taken, excluded, _ = greedy(ctx, mat, pool, conflicts(panel, hits, distinct), n_targets, max_pairs,
                                             goal, comm, crosses(sites, pool, lo, hi, comm) if cross else None, off)
            t5 = time.perf_counter()
        finally:
            mat.close()
            for s in sites:
                if s is not None:
                    s.close()
    except _lib.MpbError as exc:
        raise SystemExit("Error: %s" % exc)
    times.update(read=t1 - t0, cover=t2 - t1, background=t3 - t2, dimer=t4 - t3, greedy=t5 - t4,
                 steps=sum(1 for t in taken if t[1] > 0))
    if comm is not None and comm.rank != 0:
        return None
    write_outputs(out, pool, amp, taken, excluded, n_targets)
    return dict(taken=taken, names=pool.names, size=amp, covered=sum(t[2] for t in taken), total=n_targets)


def argsParse(argv=None):
    parser = OptionParser('Usage: %prog -r [targets.fa] -i [candidates] -f [format] -o [out_prefix]')
    ps.add_options(parser, "primer_select", "<out>.selected.tsv, <out>.candidates.tsv and <out>.selected.fa")
    parser.get_option("-f").help = "Format of primer file: xls, fa, seq or sets (get_multiPrime's candidate file)."
    parser.add_option('-k', '--max-pairs', dest='max_pairs', default=0, type="int",
                      help='Pairs to select at most, kept pairs not counted (0: no cap). Default: 0.')
    parser.add_option('--goal', dest='goal', default=1.0, type="float",
                      help='Stop when this fraction of the targets is covered (0 < goal <= 1). Default: 1.0.')
    parser.add_option('-t', '--threshold', dest='threshold', default=3.96, type="float",
                      help='Threshold of the dimer loss function (finDimer -t). Default: 3.96.')
    parser.add_option('--keep', dest='keep', default=None, help='Pairs of an existing panel, taken before any candidate.')
    parser.add_option('--keep-format', dest='keep_format', default="xls", help='Format of --keep: xls, fa or seq. '
                                                                               'Default: xls.')
    parser.add_option('--cross', dest='cross', action="store_true", default=False,
                      help='Also exclude the candidates that form a cross product with a taken pair.')
    parser.add_option('--background', dest='background', default=None,
                      help='FASTA of a background (host genome, near neighbours): a candidate with a product on it is '
                           'excluded; with --cross the cross products are searched on it too.')
    parser.add_option('--device', dest='device', default=0, type="int", help=SUPPRESS_HELP)
    args = sys.argv[1:] if argv is None else argv
    (options, rest) = parser.parse_args(args)
    fmt = options.format
    if fmt == "sets":                          # check_options knows the formats of parse_primers only
        options.format = "xls"
    options = ps.check_options(parser, options)
    options.format = fmt if fmt == "sets" else options.format
    if options.keep_format not in ("xls", "fa", "seq"):
        raise SystemExit("Error: --keep-format must be xls, fa or seq (got %s)" % options.keep_format)
    check_select(0, options.max_pairs, options.goal)
    return options


def main(argv=None, _backend=None):
    from .findimer import shard_setup
    e1 = time.time()
    options = argsParse(argv)
    cands = read_candidates(options.input, options.format)
    keep = parse_primers(options.keep, options.keep_format) if options.keep else {}
    extra, rank = shard_setup(options.device)
    res = run(options.ref, cands, options.out, options.variation, options.coordinate, options.size, options.max_pairs,
              options.goal, options.threshold, keep, options.cross, options.background, _backend=_backend, **extra)
    if "comm" in extra:
        import torch.distributed as dist
        dist.destroy_process_group()
    e2 = time.time()
    if rank == 0:
        print("INFO {} Selected: {} Covered: {}/{} Total times: {}".format(
            time.strftime("%Y-%m-%d %H:%M:%S", time.localtime(time.time())), len(res["taken"]), res["covered"],
            res["total"], round(float(e2 - e1), 2)))


if __name__ == "__main__":
    main()
