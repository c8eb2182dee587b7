"""Drop-in for scripts/finDimer.py (finDimer_V4.py / finDimer_V5_alpha.py): all-pairs primer-dimer report.

Same flags (-i -n -t -o) and output files (<out> TSV, <out>.dimer_num); rows come out in (i, j) position order as
in V5 (V4's row order depends on process scheduling).  The pair grid runs on the GPU (csrc/mpb_dimer.cu): 5-mer
prefilter over all i <= j pairs, then the reference's first-hit search on the survivors; the few hits are formatted
here with the reference's own float expressions."""
from __future__ import annotations

import argparse
import os
import time
from collections import defaultdict

import numpy as np

from . import _lib
from .dimer import dg_consts, loss_table, penalty_points
from .iupac import BASES, ORDER, sets_of

HEADERS = ["Primer_ID", "Primer seq", "Primer end", "Delta G", "Primer end length", "End (distance 1)", "End (GC)",
           "Dimer-primer_ID", "Dimer-primer seq", "End (distance 2)", "Loss"]


def parseArg(argv=None):
    parser = argparse.ArgumentParser(description="For primer dimer check")
    parser.add_argument("-i", "--input", type=str, required=True, help="input fasta primer file", metavar="<file>")
    parser.add_argument("-n", "--num", type=int, default=5, help="number of cpu process, 5 by default (accepted; the "
                                                                 "grid runs on the GPU)", metavar="<int>")
    parser.add_argument("-t", "--threshold", type=float, default=3.96,
                        help="threshold of loss function. Default: 3.96", metavar="<int>")
    parser.add_argument("-o", "--output", type=str, required=True, help="output file", metavar="<file>")
    parser.add_argument("--device", type=int, default=0, help=argparse.SUPPRESS)
    return parser.parse_args(argv)


def delta_g_plain(end: str) -> float:
    """finDimer_V4.py:171-189 for a plain (already expanded) end"""
    c = dg_consts()
    g = 0
    idx = {"A": 0, "C": 1, "G": 2, "T": 3}
    for n in range(len(end) - 1):
        g += c[idx[end[n + 1]] * 4 + idx[end[n]]]
    if end[-2:] == "TA":
        g += c[16 + idx[end[0]]] + c[16 + idx[end[-1]]] + c[20]
    else:
        g += c[16 + idx[end[0]]] + c[16 + idx[end[-1]]]
    g -= c[21] * len(end)
    half = len(end) // 2
    if len(end) % 2 == 0 and all(idx[end[i]] + idx[end[half + i]] == 3 for i in range(half)):
        g += c[22]
    return round(g, 2)


def nth_end(sets, e_idx: int, min_end: int = 5, max_end: int = 18) -> str:
    """the e_idx-th 3' end of a primer in the reference's order: suffix lengths high to low (finDimer_V4.py:193 after
    core:457-464), each suffix expanded in product order"""
    k = len(sets)
    for L in range(min(max_end, k), min_end - 1, -1):
        suffix = sets[k - L:]
        n = 1
        for s in suffix:
            n *= len(ORDER[s])
        if e_idx < n:
            out = []
            for s in reversed(suffix):
                alts = ORDER[s]
                out.append(BASES[alts[e_idx % len(alts)]])
                e_idx //= len(alts)
            return "".join(reversed(out))
        e_idx -= n
    raise IndexError("end index out of range")


def grid_hits(ctx, backend, sets_list, threshold: float, comm=None, rows_per_band: int = 0):
    """finDimer's pair grid over a primer list (base sets per primer): every (i, j >= i) that forms a dimer ->
    (hits [(i, j, order index, d2)] in (i, j) order on every rank, expansions per primer, pairs tested)"""
    eng = backend.Dimer(ctx, sets_list, 5, 18, True, loss_table(threshold), dg_consts())
    n = len(sets_list)
    rank, world = (comm.rank, comm.world) if comm else (0, 1)
    band = rows_per_band or max(1, min(n, (1 << 24) // max(1, n) * 8))
    hits = []
    tested = 0
    try:
        for b, r0 in enumerate(range(0, n, band)):
            if b % world != rank:              # row bands dealt round-robin to the ranks
                continue
            hi, hj, ho, hd, nt = eng.grid(r0, min(n, r0 + band))
            tested += nt
            hits.extend(zip(hi.tolist(), hj.tolist(), ho.tolist(), hd.tolist()))
        n_p = np.diff(eng.off_p)
    finally:
        eng.close()
    if comm and world > 1:                     # hit lists of the ranks: one variable-length gather of int64 quadruples
        flat, _ = comm.allgather_concat(np.array(hits, np.int64).reshape(-1))
        hits = sorted(tuple(int(x) for x in h) for h in flat.reshape(-1, 4))
        tested = int(comm.allreduce_sum(np.array([tested], np.int64))[0])
    return hits, n_p, tested


class Dimer(object):
    """finDimer_V4.py:127-146 constructor arguments"""

    def __init__(self, primer_file="", outfile="", threshold=3.96, nproc=10, device=0, ctx=None, comm=None,
                 _backend=None):
        self.nproc = nproc
        self.primers_file = primer_file
        self.threshold = threshold
        self.outfile = os.path.abspath(outfile)
        self.primers = self.parse_primers()
        self.primers_list = list(self.primers.keys())
        self._backend = _backend or _lib          # tests inject tests/fake_device.py
        self.ctx = ctx or self._backend.Context(device)
        self.comm = comm

    def parse_primers(self):
        """finDimer_V4.py:138-146: keyed by sequence, value = the last header seen for it"""
        primer_dict = {}
        name = ""
        with open(self.primers_file, "r") as f:
            for line in f:
                if line.startswith(">"):
                    name = line.strip()
                else:
                    primer_dict[line.strip()] = name
        return primer_dict

    def find(self, rows_per_band: int = 0):
        """all dimer rows in (i, j) order"""
        plist = self.primers_list
        sets_list = [sets_of(p.upper()) for p in plist]
        hits, n_p, self.pairs_tested = grid_hits(self.ctx, self._backend, sets_list, self.threshold, self.comm,
                                                 rows_per_band)
        rows = []
        for i, j, order, d2 in hits:
            end = nth_end(sets_list[i], order // int(n_p[j]))
            gc = end.count("G") + end.count("C")
            rows.append((self.primers[plist[i]], plist[i], end, delta_g_plain(end), len(end), 0, gc,
                         self.primers[plist[j]], plist[j], d2, penalty_points(len(end), gc, 0, d2)))
        return rows

    def run(self):
        rows = self.find()
        if self.comm and self.comm.rank != 0:
            return rows
        primer_id_sum = defaultdict(int)
        dimer_primer_id_sum = defaultdict(int)
        with open(self.outfile, "w") as fo:
            fo.write("\t".join(HEADERS) + "\n")
            for res in rows:
                primer_id_sum[res[0]] += 1
                dimer_primer_id_sum[res[7]] += 1
                fo.write("\t".join(map(str, res)) + "\n")
        with open(self.outfile + ".dimer_num", "w") as fo:
            fo.write("SeqName\tPrimer_ID\tDimer-primer_ID\tRowSum\n")
            for k in primer_id_sum.keys():
                p_id = primer_id_sum[k]
                d_id = dimer_primer_id_sum[k]
                fo.write("\t".join(map(str, [k, p_id, d_id, p_id + d_id])) + "\n")
        return rows


def shard_setup(device: int):
    """under torchrun: one rank per GPU (NCCL; MPB_DIST_BACKEND=gloo for ranks that share a GPU).  The pair grid is a set
    of independent units (SURVEY.md 8e): row bands are dealt round-robin, the sparse hit lists gathered."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1:
        return {"device": device}, 0
    import torch
    import torch.distributed as dist
    from .comm import TorchComm
    rank, local = int(os.environ["RANK"]), int(os.environ.get("LOCAL_RANK", "0"))
    backend = os.environ.get("MPB_DIST_BACKEND", "nccl")
    dev = local if backend == "nccl" else device
    if backend == "nccl":
        torch.cuda.set_device(dev)
        dist.init_process_group("nccl", device_id=torch.device("cuda", dev))
    else:
        dist.init_process_group(backend)
    return {"device": dev, "comm": TorchComm()}, rank


def main(argv=None):
    e1 = time.time()
    args = parseArg(argv)
    extra, rank = shard_setup(args.device)
    app = Dimer(primer_file=args.input, threshold=args.threshold, outfile=args.output, nproc=args.num, **extra)
    app.run()
    if "comm" in extra:
        import torch.distributed as dist
        dist.destroy_process_group()
    e2 = time.time()
    if rank == 0:
        print("INFO {} Total times: {}".format(time.strftime("%Y-%m-%d %H:%M:%S", time.localtime(time.time())),
                                               round(float(e2 - e1), 2)))


if __name__ == "__main__":
    main()
