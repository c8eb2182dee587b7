"""Host side of the degenerate-primer candidate scan: a drop-in for scripts/multiPrime-core.py (V20).

`NN_degenerate` keeps the reference's constructor arguments, `run()` and output files (core:343-365,
1133-1180).  All per-sequence work — window extraction with gap patching, haplotype counting, base / dinucleotide
tensors, the mismatch scan, Tm — runs in libmpb200.so on an H100; this module holds the per-window control logic
(gates, seeds, the NN-array refinement walk, filters, writers), which only ever touches O(k) numbers per window.

There is no CPU fallback: constructing NN_degenerate without a CUDA device raises.
"""
from __future__ import annotations

import json
import math
import os
import sys
import time
from statistics import mean

import numpy as np

from . import _lib
from .comm import NoComm
from .iupac import BASES, CODE_CHARS, CHAR_CODE, allow_masks, expand_array, expand_keys, expand_strings, primer_string, rc_sets

TSV_HEADER = ["Position", "Entropy of cover (bit)", "Entropy of total (bit)", "Optimal_primer",
              "primer_degenerate_number", "nonsense_primer_number", "Optimal_coverage", "Mis-F-coverage",
              "Mis-R-coverage", "Tm", "Information"]


# ----------------------------------------------------------------------------------------------------------
# input
# ----------------------------------------------------------------------------------------------------------
def _byte_table() -> bytes:
    t = bytearray(256)
    for ch, code in CHAR_CODE.items():
        if ch in "ACGTRYMKSWHBVD":              # core:453: everything else (N included) becomes a gap
            t[ord(ch)] = code
            t[ord(ch.lower())] = code
    return bytes(t)


_BYTE_TABLE = _byte_table()


def parse_msa(path: str):
    """core:441-455 parse_seq -> (ids, codes uint8 [n_seq, n_col] of 4-bit base sets, lens int32)"""
    order: dict[str, list] = {}
    cur = None
    with open(path, "rb") as fh:
        for line in fh:
            if line.startswith(b"#"):
                continue
            if line.startswith(b">"):
                cur = line.decode().strip().split(" ")[0]
            else:
                order.setdefault(cur, []).append(line.strip().translate(_BYTE_TABLE))
    ids = list(order.keys())
    rows = [b"".join(parts) for parts in order.values()]
    lens = np.array([len(r) for r in rows], dtype=np.int32)
    n_col = int(lens.max()) if len(rows) else 0
    if len(rows) and (lens == n_col).all():
        codes = np.frombuffer(b"".join(rows), dtype=np.uint8).reshape(len(rows), n_col)
    else:
        codes = np.zeros((len(rows), n_col), dtype=np.uint8)
        for i, r in enumerate(rows):
            codes[i, :len(r)] = np.frombuffer(r, dtype=np.uint8)
    return ids, codes, lens


def pack4(codes: np.ndarray) -> np.ndarray:
    """two cells per byte, low nibble = even column"""
    n, L = codes.shape
    if L % 2:
        codes = np.concatenate([codes, np.zeros((n, 1), np.uint8)], axis=1)
    return (codes[:, 0::2] | (codes[:, 1::2] << 4)).astype(np.uint8)


def strict_masks(coordinate: str, k: int):
    """core:1091-1101 get_Y as bit masks over 0-based primer positions (indices >= k never match anything)"""
    f = r = 0
    for tok in coordinate.split(","):
        y = int(tok.strip())
        fi, ri = (y, k - y) if y > 0 else (k + y + 1, -y + 1)
        if 0 <= fi < k:
            f |= 1 << fi
        if 0 <= ri < k:
            r |= 1 << ri
    return f, r


# ----------------------------------------------------------------------------------------------------------
# scalar pieces evaluated per window on the host
# ----------------------------------------------------------------------------------------------------------
def _tm_consts():
    """the sequence-independent terms of core:293-335, spelled as the reference spells them"""
    primer_concentration, Mo, Di, dNTP = 100, 50, 1.5, 0.25
    free_divalent = (Di - dNTP) / 1000.0
    a = 3.92 * pow(10, -5) * (0.843 - (0.352 * math.sqrt(Mo / 1000.0) * math.log(Mo / 1000.0, math.e)))
    b = - 9.11 * pow(10, -6)
    correction = a + (b * math.log(free_divalent, math.e))          # core:323 (the rest of Eq 16 is dead code)
    c4 = 1.9872 * math.log(primer_concentration / (4 * pow(10, 9)), math.e)
    c1 = 1.9872 * math.log(primer_concentration / (1 * pow(10, 9)), math.e)
    return c4, c1, correction


TM_CONSTS = _tm_consts()


# ---- filters (core:387-416, 507-521) on base-set lists, no expansion ------------------------------------
def _repeat_patterns():
    pats = set()
    for i in range(4):
        pats.add((i,) * 4)
        for j in range(4):
            if i != j:
                pats.add((i, j) * 4)
            for kk in range(4):
                if i != j and j != kk:
                    pats.add((i, j, kk) * 3)
    return sorted(pats)


_REPEATS = _repeat_patterns()


def gc_content(sets) -> float:
    """core:401-407: mean over expansions of round(gc/len, 3), rounded to 2 — via the GC-count distribution"""
    k = len(sets)
    dist = [1]                                    # dist[g] = number of expansions of the prefix with g G/C
    for s in sets:
        n_gc = ((s >> 1) & 1) + ((s >> 2) & 1)
        n_at = (s & 1) + ((s >> 3) & 1)
        new = [0] * (len(dist) + 1)
        for g, m in enumerate(dist):
            new[g] += m * n_at
            new[g + 1] += m * n_gc
        dist = new
    total = sum(dist)
    acc = 0
    for g, m in enumerate(dist):
        if m:
            acc += m * int(round(g / k, 3) * 1152921504606846976.0)   # exact: round(g/k, 3) is 0 or >= 2^-8
    return round(acc / (total << 60), 2)                               # statistics.mean: exact rational mean


def has_repeat(sets) -> bool:
    """core:410-416: some expansion contains XXXX, (XY)x4 or (XYZ)x3"""
    k = len(sets)
    allow = allow_masks(sets)
    for pat in _REPEATS:
        n = len(pat)
        if n > k:
            continue
        hit = (1 << (k - n + 1)) - 1
        for t, b in enumerate(pat):
            hit &= allow[b] >> t
            if not hit:
                break
        if hit:
            return True
    return False


def has_hairpin(sets, distance: int) -> bool:
    """core:387-398: a 5-mer whose reverse complement can occur at least `distance` bases downstream"""
    k = len(sets)
    n = 0
    while n <= k - 5 - 5 - distance:
        target = rc_sets(sets[n:n + 5])
        tail0 = n + 5 + distance
        for o in range(tail0, k - 5 + 1):
            if all(target[t] & sets[o + t] for t in range(5)):
                return True
        n += 1
    return False


def information(sets, gc_lo: float, gc_hi: float, distance: int):
    """core:507-521 primer_pre_filter"""
    notes = []
    gc = gc_content(sets)
    if not gc_lo <= gc <= gc_hi:
        notes.append("GC_out_of_range (" + str(gc) + ")")
    if has_repeat(sets):
        notes.append("di_nucleotide")
    if has_hairpin(sets, distance):
        notes.append("hairpin")
    return gc if not notes else "|".join(notes)


class NN_degenerate(object):
    """Drop-in for the reference class of the same name (core:342-365); same keyword arguments.

    Extra keyword arguments (not in the reference): device, windows_per_batch, sidecars."""

    def __init__(self, seq_file, primer_length=18, coverage=0.8, number_of_dege_bases=18, score_of_dege_bases=1000,
                 product_len=250, position="2,-1", variation=2, raw_entropy_threshold=3.6, distance=4, GC="0.4,0.6",
                 nproc=10, outfile="", device=0, windows_per_batch=0, sidecars=True, alignment=None, packed=None,
                 stream=None, comm=None, row0=0, want_trace=True, keep_bits=False, rows_on_rank0_only=False,
                 sidecar_format="auto", _backend=None):
        self.primer_length = primer_length
        self.coverage = coverage
        self.number_of_dege_bases = number_of_dege_bases
        self.score_of_dege_bases = score_of_dege_bases
        self.product = product_len
        self.position = position
        self.variation = variation
        self.distance = distance
        self.GC = GC.split(",")
        self.nproc = nproc                      # accepted and ignored, as in the reference (core:1143)
        self.raw_entropy_threshold = raw_entropy_threshold
        self.outfile = outfile
        self.sidecars = sidecars
        self.want_trace = want_trace            # record the primers handed to mis_primer_check (the tests compare them)
        self.keep_bits = keep_bits              # keep the per-sequence F / R / gap bit vectors of every row (pairing)
        self.bit_vectors = []
        self.rows_on_rank0_only = rows_on_rank0_only   # sharded runs: the replicated row assembly on rank 0 only
        self.sidecar_format = sidecar_format    # run(): "json" (the reference's two files), "bits", "auto" by size
        self.windows_per_batch = windows_per_batch
        if not 3 <= primer_length <= _lib.MAX_K:
            raise ValueError("primer length must be within 3..%d" % _lib.MAX_K)
        t_init = [time.perf_counter()]
        self.init_ms = {}

        def lap(name):
            now = time.perf_counter()
            self.init_ms[name] = 1000 * (now - t_init[0])
            t_init[0] = now
        self.fmask, self.rmask = strict_masks(position, primer_length)
        if packed is not None:                   # (ids, nibble-packed rows, n_col, lens): already in upload format
            self.ids, packed4, self.n_col, lens = packed
            self._codes = None
        else:
            self.ids, codes, lens = alignment if alignment is not None else parse_msa(seq_file)
            self.n_col = codes.shape[1]
            self._codes = codes
            packed4 = pack4(codes)
        self._row_cache = {}
        self._packed4 = packed4                 # host copy: only read for the rare IUPAC-in-gap-row side-file entries
        self.comm = comm or NoComm()            # sequence shards: this process holds rows [row0, row0 + n_local)
        self.row0 = row0
        self.n_local = len(self.ids)
        self.total_sequence_number = int(self.comm.allreduce_sum(np.array([self.n_local], np.int64))[0])
        self.lens = lens if lens is not None else np.full(len(self.ids), self.n_col, np.int32)
        backend = _backend or _lib                # tests inject tests/fake_device.py to exercise the host logic
        self.ctx = backend.Context.shared(device, stream) if hasattr(backend.Context, "shared") else \
            backend.Context(device, stream)
        self.msa = backend.Msa(self.ctx, packed4, len(self.ids), self.n_col,
                               lens=None if (self.lens == self.n_col).all() else self.lens)
        if row0:
            self.msa.set_row0(row0)
        # sequence shards, one GPU per rank: the walk sums its count vectors over NVLink peer memory (mpb_peer_*)
        self.peer = None
        if self.comm.world > 1 and getattr(self.comm, "peer_ok", False) and hasattr(backend, "Peer") \
                and os.environ.get("MPB_PEER", "1") != "0":
            self.peer = backend.Peer.of(self.ctx, self.comm)
        lap("upload")
        self.position_list = self.seq_attribute()
        lap("region")
        self.start_position, self.stop_position, self.length = self.position_list
        self.entropy_threshold = self.entropy_threshold_adjust(self.length)
        self.stats = {"windows": 0, "accepted": 0, "scan_calls": 0, "evals": 0, "candidates": 0}

    # -- core:617-649 -------------------------------------------------------------------------------------
    def seq_attribute(self):
        lead_hist, rstrip_hist = self.msa.seq_attr_hist()
        if self.comm.world > 1:                 # the quantiles are over all sequences: shards add their histograms
            lead_hist = self.comm.allreduce_sum(lead_hist)
            rstrip_hist = self.comm.allreduce_sum(rstrip_hist)
        # np.quantile(x, q, "higher" / "lower") = sorted(x)[ceil / floor((n - 1) * q)]: an order statistic, read off the
        # cumulative histogram
        vidx = (self.total_sequence_number - 1) * self.coverage
        start = int(np.searchsorted(np.cumsum(lead_hist), math.ceil(vidx), side="right"))
        stop = int(np.searchsorted(np.cumsum(rstrip_hist), math.floor(vidx), side="right"))
        if stop - start < int(self.product):
            print("Error: max length of PCR product is shorter than the default min Product length with {} "
                  "coverage! Non candidate primers !!!".format(self.coverage))
            sys.exit(1)
        return [start, stop, stop - start]

    def entropy_threshold_adjust(self, length):
        if length < 5000:
            return self.raw_entropy_threshold
        if length < 10000:
            return self.raw_entropy_threshold * 0.95
        return self.raw_entropy_threshold * 0.9

    # -- entropy (core:602-614) ----------------------------------------------------------------------------
    def _exception_records(self, hist) -> np.ndarray:
        """gap rows that hold IUPAC cells are not in the device table (their raw k-mer needs 4 bits per cell): one record
        (first order, count, window, raw cells 0..14, raw cells 15..) per such (window, local sequence), cut from the
        host copy; the k 4-bit cells travel folded into two integers"""
        k = self.primer_length
        exc_w, exc_s = self._exceptions(hist)
        rec = np.zeros((len(exc_w), 5), np.int64)
        if len(exc_w):
            exc_pos = np.asarray(hist.win_pos)[exc_w]
            cells, got = _lib.window_cells(self._packed4, self.lens, self.n_col, k, exc_s, exc_pos)
            if (got < k).any():
                raise ValueError("a sequence is too short to supply a %d-mer at window %d"
                                 % (k, int(exc_pos[np.argmax(got < k)])))
            cells = cells.astype(np.int64)
            rec[:, 0] = (self.row0 + exc_s.astype(np.int64)) << 16
            rec[:, 1] = 1
            rec[:, 2] = exc_w
            for j in range(k):
                rec[:, 3 if j < 15 else 4] |= cells[:, j] << (4 * (j if j < 15 else j - 15))
        return rec

    def _group_exception_records(self, rec) -> dict:
        """{window: [(first order, count)]}: the records grouped by (window, raw k-mer)"""
        cache = {}
        if len(rec):
            lo, hi = rec[:, 3], rec[:, 4]                  # rows sorted by (window, raw k-mer), runs reduced
            order = np.lexsort((lo, hi, rec[:, 2]))
            w_s, lo_s, hi_s = rec[order, 2], lo[order], hi[order]
            new_run = np.ones(len(rec), bool)
            new_run[1:] = (w_s[1:] != w_s[:-1]) | (lo_s[1:] != lo_s[:-1]) | (hi_s[1:] != hi_s[:-1])
            starts = np.nonzero(new_run)[0]
            first = np.minimum.reduceat(rec[order, 0], starts)
            count = np.add.reduceat(rec[order, 1], starts)
            win = w_s[starts]
            cuts = np.nonzero(np.diff(win))[0] + 1
            for a, b in zip(np.concatenate([[0], cuts]).tolist(), np.concatenate([cuts, [len(win)]]).tolist()):
                cache[int(win[a])] = list(zip(first[a:b].tolist(), count[a:b].tolist()))
        return cache

    def _iupac_gap_groups(self, hist, wi):
        """[(first order, count)] of the gap rows of window wi that hold IUPAC cells (a sharded run fills the cache in
        _exchange, where the shards' records travel with the window counters)"""
        cache = getattr(hist, "_iupac_groups", None)
        if cache is None:
            cache = hist._iupac_groups = self._group_exception_records(self._exception_records(hist))
            ws = [w for w, groups in cache.items() for _ in groups]
            cs = [c for groups in cache.values() for _, c in groups]
            hist._iupac_sums = (np.array(ws, np.int64), np.array(cs, np.int64))
        return cache.get(wi, [])

    def _entropy_exact(self, table, ti, wi, n_unique, hist=None):
        """the reference's left-to-right float sums (core:602-614), over the table dumped in first-seen order.
        table / ti: the handle holding the complete table of the window and its index there; wi: the window's index in
        the batch (hist: the local handle that carries the exception rows, when it is another one than `table`)."""
        k, v = self.primer_length, self.variation
        keys, cnt, first = table.dump(ti, int(n_unique) + 8)
        is_gap = np.zeros(len(keys), bool)
        b5 = keys >= np.uint64(_lib.KEY_BASE5)
        if b5.any():
            x = (keys[b5] - np.uint64(_lib.KEY_BASE5)).astype(np.uint64)
            g = np.zeros(len(x), np.int64)
            for _ in range(k):
                g += (x % np.uint64(5)) == np.uint64(4)
                x //= np.uint64(5)
            is_gap[b5] = g > v
        cover = cnt[~is_gap].tolist()                                   # dump() is sorted by first-seen order
        gaps = list(zip(first[is_gap].tolist(), cnt[is_gap].tolist())) + self._iupac_gap_groups(hist or table, wi)
        gaps.sort()
        gap_n = sum(c for _, c in gaps)
        cover_number = self.total_sequence_number - gap_n
        tot = cover_number + gap_n
        term_c, term_t = {}, {}
        for c in set(cover):
            term_c[c] = (c / cover_number) * math.log((c / cover_number), 2)
        for c in set(cover) | {c for _, c in gaps}:
            term_t[c] = (c / tot) * math.log((c / tot), 2)
        c_bit = 0
        t_bit = 0
        for c in cover:                  # plain left-to-right adds (the builtin sum() is compensated since 3.12)
            c_bit += term_c[c]
            t_bit += term_t[c]
        for _, c in gaps:
            t_bit += term_t[c]
        return round(-c_bit, 2), round(-t_bit, 2)

    def _exceptions(self, hist):
        if getattr(hist, "_exc", None) is None:
            hist._exc = hist.exceptions()
        return hist._exc

    def _window_cells(self, s: int, p: int) -> bytes:
        """core:666-687 for one (sequence, window) on the host copy; only used for IUPAC-holding gap rows"""
        k = self.primer_length
        row = self._row_cache.get(s)
        if row is None:
            if self._codes is not None:
                row = self._codes[s, :self.lens[s]].tobytes()
            else:
                pk = self._packed4[s]
                cells = np.empty(pk.shape[0] * 2, np.uint8)
                cells[0::2] = pk & 15
                cells[1::2] = pk >> 4
                row = cells[:self.lens[s]].tobytes()
            if len(self._row_cache) < 200000:
                self._row_cache[s] = row
        gap = b"\x00"
        w = row[p:p + k]
        if w != gap * k:
            if w.startswith(gap):
                body = w.lstrip(gap)
                g = len(w) - len(body)
                left = row[0:p].replace(gap, b"")
                if len(left) >= g:
                    w = left[len(left) - g:] + body
            if w.endswith(gap):
                body = w.rstrip(gap)
                g = len(w) - len(body)
                right = row[p + k:].replace(gap, b"")
                if len(right) >= g:
                    w = body + right[0:g]
        if len(w) < k:
            g = k - len(w)
            left = row[0:p].replace(gap, b"")
            if len(left) >= g:
                w = left[len(left) - g:] + w
        return w

    def _table_log2cap(self, k: int, n: int) -> int:
        """log2 of the slots per haplotype table holding the haplotypes of n sequences, 0 = the library default (two
        slots per sequence).
        The windows that reach the tables passed the prefilter: the entropy of their 65536 coarse bins is at most the
        gate, so a fraction x of items that are (nearly) alone in their bin costs x * (16 + log2(1/x)) bits and x stays
        below thr / 16-ish (0.2 for the default 3.6 bits) — distinct haplotypes are a fifth of the sequences at most,
        in practice far fewer.  Tables of N / 2 slots (load <= 0.4) are a quarter of the default.  A table that fills
        up anyway reports MPB_EOVERFLOW and is rebuilt with doubled capacity (_lib.Hist for the local build,
        _exchange for the owner tables of a sharded run)."""
        if k < 8 or n < (1 << 17) or self.entropy_threshold > 4.0:
            return 0
        return max(10, int(math.ceil(math.log2(n / 2))))

    # -- the window pipeline --------------------------------------------------------------------------------
    def design(self, positions):
        """Run the per-window algorithm (core:651-858) for the given window start columns.
        Returns a list of records {row, non_cov, gap_ids, trace} (rejected windows are absent)."""
        positions = [int(p) for p in positions]
        self.bit_vectors = []
        if not positions:
            return []
        per_batch = min(65535, self.windows_per_batch or _default_batch(self.n_local))
        out = []
        for b0 in range(0, len(positions), per_batch):
            out.extend(self._design_batch(positions[b0:b0 + per_batch]))
        return out

    def _design_batch(self, positions):
        k, v, N = self.primer_length, self.variation, self.total_sequence_number
        comm = self.comm
        self.stats["windows"] += len(positions)
        ph = self.stats.setdefault("phase_ms", {})
        tick = [time.perf_counter()]

        def lap(name):
            now = time.perf_counter()
            ph[name] = ph.get(name, 0.0) + 1000 * (now - tick[0])
            tick[0] = now

        # entropy prefilter: windows whose coarse-grained entropy bound is above the gate never get a table
        if k >= 8:
            if self.n_local > 0:
                s0, s1 = self.msa.prefilter(k, v, positions)
                bound = (s0 * math.log2(self.n_local) - s1) / N     # shards: size-weighted (concavity of the entropy)
            else:
                bound = np.zeros(len(positions))
            if comm.world > 1:
                bound = comm.allreduce_sum(bound)
            keep_pos = bound <= self.entropy_threshold + 0.006
        else:                                                    # very short primers: keep every window
            keep_pos = np.ones(len(positions), bool)
        self.stats["prefiltered"] = self.stats.get("prefiltered", 0) + int((~keep_pos).sum())
        positions = [p for p, kp in zip(positions, keep_pos.tolist()) if kp]
        lap("prefilter")
        if not positions:
            return []
        # sequence shards: rank r OWNS the windows with (batch index mod world) == r
        owner = (np.arange(len(positions)) % comm.world).astype(np.int32)
        with self.msa.hist(k, v, positions, self._table_log2cap(k, self.n_local)) as hist:
            lap("hist_build")
            own = None
            try:
                if comm.world > 1:
                    st, own, mine = self._exchange(hist, positions, owner)
                    lap("exchange")
                else:
                    st, mine = hist.stats(), None        # tensors follow for the windows that pass the gates only
                    lap("summary")
                out = self._gates_walk_finish(hist, own, mine, owner, st, positions, lap)
            finally:
                if own is not None:
                    own.close()
        lap("free")
        return out

    def _gates_walk_finish(self, hist, own, mine, owner, st, positions, lap):
        k, v, N = self.primer_length, self.variation, self.total_sequence_number
        comm = self.comm
        gap_n = st["gap_n"]
        # core:713 `round(gap_n / N, 2) >= 1 - coverage`: exact for all but ratios on a rounding tie
        ratio = gap_n / N
        gap_fail = np.round(ratio, 2) >= (1 - self.coverage)
        for wi in np.nonzero(np.abs((ratio * 100) % 1 - 0.5) < 1e-6)[0]:
            gap_fail[wi] = round(int(gap_n[wi]) / N, 2) >= (1 - self.coverage)
        alive = ~gap_fail & (st["nuniq"][:, 0] >= 1)                      # core:716
        accepted = []                          # (batch index, position, cBit, tBit, cover_number, has gap-free)
        for wi, ent in self._entropies(hist, own, mine, owner, st, positions, alive):
            accepted.append((wi, positions[wi], ent[0], ent[1], N - int(gap_n[wi]), bool(st["nuniq"][wi, 2] > 0)))
        lap("gates")
        if not accepted:
            return []
        if "freq" in st:                       # sharded run: the owners' tensors came with the statistics
            freq, nn = st["freq"], st["nn"]
        else:
            sel = np.zeros(len(positions), np.uint8)
            sel[[a[0] for a in accepted]] = 1
            freq, nn = hist.tensors(sel)
            lap("tensors")
        acc_w = np.array([a[0] for a in accepted], np.int64)                   # core:736-740, all windows at once
        fa = freq[acc_w]
        ok = ~((fa.sum(axis=2) == 0).any(axis=1) | (fa.sum(axis=1) == 0).any(axis=1))
        keep = [a for a, o in zip(accepted, ok.tolist()) if o]
        if not keep:
            return []
        wis = np.array([a[0] for a in keep], np.int32)
        mm_key = np.where(np.array([a[5] for a in keep]), st["mm_key"][wis], np.uint64(_lib.KEY_EMPTY))
        sharded = comm.world > 1
        res = hist.walk(self.number_of_dege_bases, self.score_of_dege_bases, self.fmask, self.rmask, wis,
                        np.array([a[4] for a in keep], np.int64), mm_key,
                        freq=freq[wis] if sharded else None, nn=nn[wis].reshape(len(keep), k - 1, 16) if sharded else None,
                        comm=comm if sharded else None, want_trace=self.want_trace,
                        **({"peer": self.peer} if self.peer is not None else {}))
        lap("walk")
        self.stats["scan_calls"] += int(res["stats"][0])
        self.stats["candidates"] += int(res["stats"][1])
        self.stats["evals"] += int(res["stats"][2]) * N
        out = self._finish(hist, own, mine, owner, keep, res)
        lap("finish")
        return out

    EXC_INLINE = 2048          # exception records carried by the counter gather of a sharded batch (80 KB per rank)

    def _exchange(self, hist, positions, owner):
        """Sequence-sharded run (SURVEY.md 8e): every per-window quantity is a sum over sequences.  Gap counters are
        summed; the haplotype entries of every window travel to the window's OWNER (one all-to-all), which merges
        them into its own table, takes the window statistics and tensors, and the small per-window results are
        all-gathered: every rank ends up with the same `st` for all windows and takes identical decisions, while the
        table work is divided by the world size.  Two host collectives (counters + exception rows; per-window
        results) and one device all-to-all per array."""
        comm, N, k, v = self.comm, self.total_sequence_number, self.primer_length, self.variation
        world, rank, nw = comm.world, comm.rank, len(positions)
        ph = self.stats.setdefault("phase_ms", {})
        tick = [time.perf_counter()]

        def lap(name):
            now = time.perf_counter()
            ph[name] = ph.get(name, 0.0) + 1000 * (now - tick[0])
            tick[0] = now

        gap_local, iupac_local, n_ent = hist.counts()
        # collective 1: per-window counters of every shard and its gap rows holding IUPAC cells (5 integers per record,
        # EXC_INLINE of them ride along; only a shard with more triggers a second, padded gather)
        exc = self._exception_records(hist)
        inline = np.zeros((self.EXC_INLINE, 5), np.int64)
        inline[:min(len(exc), self.EXC_INLINE)] = exc[:self.EXC_INLINE]
        head = np.concatenate([gap_local, iupac_local, n_ent, [len(exc)], inline.reshape(-1)]).astype(np.int64)
        heads_flat = comm.allgather_fixed(head)
        heads = heads_flat[:, :3 * nw].reshape(world, 3, nw)
        n_exc = heads_flat[:, 3 * nw]
        exc_in = heads_flat[:, 3 * nw + 1:].reshape(world, self.EXC_INLINE, 5)
        parts = [exc_in[r, :min(int(n_exc[r]), self.EXC_INLINE)] for r in range(world)]
        if int(n_exc.max()) > self.EXC_INLINE:
            pad = np.zeros((int(n_exc.max()) - self.EXC_INLINE, 5), np.int64)
            pad[:max(0, len(exc) - self.EXC_INLINE)] = exc[self.EXC_INLINE:]
            exc_all = comm.allgather_fixed(pad)
            parts += [exc_all[r, :max(0, int(n_exc[r]) - self.EXC_INLINE)] for r in range(world)]
        exc = np.concatenate(parts) if parts else exc
        # only a window's owner needs them (entropy of its window, exact replay): the others drop them unsorted
        exc = exc[owner[exc[:, 2]] == rank] if len(exc) else exc
        hist._iupac_groups = self._group_exception_records(exc)
        gap_n, iupac_gap = heads[:, 0].sum(axis=0), heads[:, 1].sum(axis=0)
        lap("x_counters")
        gap_fail = np.array([round(int(g) / N, 2) >= (1 - self.coverage) for g in gap_n])
        travel = ~gap_fail
        sizes_all = np.where(travel[None, :], heads[:, 2], 0).astype(np.int64)     # world x nw entry counts
        mine = np.nonzero(owner == rank)[0]                                        # my windows (ascending batch index)
        order = np.concatenate([np.nonzero(owner == r)[0] for r in range(world)])   # owner-major export order
        send_counts = np.array([int(sizes_all[rank, owner == r].sum()) for r in range(world)], np.int64)
        recv_counts = sizes_all[:, mine].sum(axis=1).astype(np.int64)
        on_gpu = getattr(comm, "on_gpu", False) and hasattr(hist, "export_dev")
        if on_gpu:                                 # entries stay in HBM: export -> NCCL all-to-all -> merge
            keys, cnt, first = hist.export_at(order, sizes_all[rank, order], comm)
            rk, rc, rf = (comm.alltoall_dev(t, send_counts, recv_counts) for t in (keys, cnt, first))
        else:
            keys, cnt, first = hist.export_at(order, sizes_all[rank, order])
            rk, rc, rf = (comm.alltoall(a, send_counts, recv_counts) for a in (keys, cnt, first))
        lap("x_alltoall")
        # segment offsets of the received entries: source rank major, my windows inside
        seg = np.concatenate([[0], np.cumsum(sizes_all[:, mine].reshape(-1))]).astype(np.int64)
        my_pos = [positions[i] for i in mine]
        # owner tables: the entries arriving for a window bound its distinct haplotypes, so twice the largest arrival
        # (load <= 0.5) is room enough, and far less to clear than a table sized by the sequence count
        most = int(sizes_all[:, mine].sum(axis=0).max()) if len(mine) else 0
        log2cap = max(8, int(math.ceil(math.log2(2 * most + 64))))
        per = int(np.ceil(nw / world))
        fields = [("ent", 4, np.float64), ("nuniq", 3, np.int64), ("mm_key", 1, np.uint64), ("mm_cnt", 1, np.int64),
                  ("mm_first", 1, np.uint64), ("freq", 4 * k, np.int64), ("nn", 16 * (k - 1), np.int64)]
        width = 1 + sum(f[1] for f in fields)
        own = None
        while True:
            rec = np.zeros((per, width), np.int64)
            if len(mine):
                own = self.msa.hist(k, v, my_pos, log2cap, empty=True)
                try:
                    own.merge_segments(seg, rk, rc, rf)
                    own.add_counts(gap_n[mine], iupac_gap[mine])
                    st_own = own.summary()
                    if hist._iupac_groups:                      # gap rows holding IUPAC cells are not table entries
                        slot = {int(wi): j for j, wi in enumerate(mine.tolist())}
                        gj = np.array([slot[w] for w, groups in hist._iupac_groups.items() for _ in groups], np.int64)
                        gc_f = np.array([c for groups in hist._iupac_groups.values() for _, c in groups], np.float64)
                        st_own["ent"][:, 2] += np.bincount(gj, weights=gc_f, minlength=len(mine))
                        st_own["ent"][:, 3] += np.bincount(gj, weights=gc_f * np.log2(gc_f), minlength=len(mine))
                    c0 = 1
                    for name, w, dt in fields:
                        rec[:len(mine), c0:c0 + w] = np.ascontiguousarray(st_own[name]).reshape(len(mine), w).view(np.int64)
                        c0 += w
                except _lib.MpbError as exc:
                    if exc.code != -4:
                        raise
                    rec[:, 0] = 1              # a full table on one rank is a collective event (column 0 = failed)
            lap("x_merge_summary")
            # collective 2: the per-window results of every owner (fixed-size records, padded to the maximum)
            rec_all = comm.allgather_fixed(rec)
            lap("x_results")
            if not rec_all[:, :, 0].any():
                break
            if own is not None:                # everybody rebuilds with doubled owner tables
                own.close()
                own = None
            log2cap += 1
        st = {}
        c0 = 1
        for name, w, dt in fields:
            full = np.zeros((nw, w), dt)
            for r in range(world):
                idx = np.nonzero(owner == r)[0]
                full[idx] = np.ascontiguousarray(rec_all[r, :len(idx), c0:c0 + w]).view(dt)
            st[name] = full.reshape(nw) if w == 1 else full
            c0 += w
        st["freq"] = st["freq"].reshape(nw, 4, k)
        st["nn"] = st["nn"].reshape(nw, k - 1, 4, 4)
        st["gap_n"] = gap_n
        st["n_iupac_gap"] = iupac_gap
        st["ent_complete"] = True              # the owners added the IUPAC gap rows to their windows' sums
        # windows that failed the gap gate did not travel: their (empty) statistics must not pass a later gate
        st["nuniq"][gap_fail] = 0
        return st, own, mine

    def _entropies(self, hist, own, mine, owner, st, positions, alive):
        """(window index, (cBit, tBit)) of the windows that pass the entropy gate (core:722-726), rounded as the
        reference rounds them.  The device sums use another summation order than the reference: whenever that could
        change a rounded digit or the gate, the table is dumped and the reference's float sum replayed (by the window's
        owner in a sharded run; the result is shared)."""
        N = self.total_sequence_number
        thr = self.entropy_threshold
        comm = self.comm
        ent = st["ent"].astype(np.float64).copy()
        if not st.get("ent_complete") and (alive & (st["n_iupac_gap"] > 0)).any():
            self._iupac_gap_groups(hist, -1)                   # gap rows holding IUPAC cells: fills the cache
            gw, gc_ = hist._iupac_sums                         # (window, count) of every group of equal raw k-mers
            if len(gw):
                gc_f = gc_.astype(np.float64)
                ent[:, 2] += np.bincount(gw, weights=gc_f, minlength=len(ent))
                ent[:, 3] += np.bincount(gw, weights=gc_f * np.log2(gc_f), minlength=len(ent))
        cover_number = (N - st["gap_n"]).astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            c_raw = -(ent[:, 1] - ent[:, 0] * np.log2(cover_number)) / cover_number
            t_raw = -((ent[:, 1] - ent[:, 0] * math.log2(N)) + (ent[:, 3] - ent[:, 2] * math.log2(N))) / N
        tie = lambda x: np.abs((x * 100.0) % 1.0 - 0.5) < 1e-6
        exact = tie(c_raw) | tie(t_raw) | (np.abs(t_raw - thr) < 1e-6) | (np.abs(c_raw) < 1e-9) | (np.abs(t_raw) < 1e-9)
        # (an exact zero prints as "-0.0" in the reference: round(-0.0, 2); that is left to the replay too)
        cand = np.nonzero(alive & (exact | ~(t_raw > thr + 0.006)))[0].tolist()
        replay = {}
        need = [wi for wi in cand if exact[wi]]
        if need:
            vals = np.zeros((len(need), 2), np.float64)
            for j, wi in enumerate(need):
                if comm.world == 1:
                    vals[j] = self._entropy_exact(hist, wi, wi, int(st["nuniq"][wi, 0] + st["nuniq"][wi, 1]))
                elif owner[wi] == comm.rank:
                    vals[j] = self._entropy_exact(own, int(np.searchsorted(mine, wi)), wi,
                                                  int(st["nuniq"][wi, 0] + st["nuniq"][wi, 1]), hist)
            if comm.world > 1:          # only the owner holds the merged table; -0.0 survives as a bit pattern
                vals = comm.allreduce_sum(vals.view(np.int64)).view(np.float64)
            replay = {wi: (float(vals[j, 0]), float(vals[j, 1])) for j, wi in enumerate(need)}
        out = []
        for wi, c_x, t_x, ex in zip(cand, c_raw[cand].tolist(), t_raw[cand].tolist(), exact[cand].tolist()):
            c_bit, t_bit = replay[wi] if ex else (round(c_x, 2), round(t_x, 2))
            if not t_bit > thr:                                               # core:723
                out.append((wi, (c_bit, t_bit)))
        return out

    # -- rows, filters, side files ----------------------------------------------------------------------------
    def _finish(self, hist, own, mine, owner, keep, res):
        """core:846-858 row assembly for the windows that went through the walk"""
        k, v, N = self.primer_length, self.variation, self.total_sequence_number
        gc_lo, gc_hi = float(self.GC[0]), float(self.GC[1])
        n = len(keep)
        ph = self.stats.setdefault("phase_ms", {})
        tick = [time.perf_counter()]

        def lap(name):
            now = time.perf_counter()
            ph[name] = ph.get(name, 0.0) + 1000 * (now - tick[0])
            tick[0] = now

        sets_arr = res["sets"]
        sets_list = [row[:k].tolist() for row in sets_arr]
        wis = np.array([a[0] for a in keep], np.int32)
        pos = np.array([a[1] for a in keep], np.int32)
        place = np.uint32(1) << np.arange(k, dtype=np.uint32)            # allow_masks() of every primer at once
        allow = np.stack([(((sets_arr[:, :k] >> b) & 1).astype(np.uint32) * place).sum(axis=1, dtype=np.uint32)
                          for b in range(4)], axis=1)
        # perfect coverage of the chosen primer is already known from the walk (the last candidate scanned for the
        # track IS the final primer); a final scan pass is only needed for the per-sequence non-cover bits
        bits = None
        if self.sidecars or self.keep_bits:
            # per-sequence F / R non-cover and gap-row bits of the final primers: to the host for the JSON side files,
            # left in HBM when only the pairing step (pairing.py) consumes them
            on_dev = self.keep_bits and not self.sidecars and hasattr(self.ctx, "h")
            _, bits = hist.cscan(self.fmask, self.rmask, _lib.make_cands(wis, allow), bits_slot=np.arange(n, dtype=np.int32),
                                 bits_out="device" if on_dev else None)
            self.stats["scan_calls"] += 1
            if self.keep_bits:
                self.bit_vectors.append((pos.copy(), bits))
        perfect = res["counts"][:, 4]
        lap("fin_scan")
        if self.comm.world == 1:
            distinct = hist.match(wis, allow)
        else:                          # the merged table of a window lives on its owner
            distinct = np.zeros(n, np.int64)
            sel = np.nonzero(owner[wis] == self.comm.rank)[0]
            if len(sel):
                distinct[sel] = own.match(np.searchsorted(mine, wis[sel]).astype(np.int32), allow[sel])
            distinct = self.comm.allreduce_sum(distinct)
        lap("fin_match")
        world, rank = self.comm.world, self.comm.rank
        if world == 1:
            tm_avg, gc, flags, deg, ndeg = self._primer_props(sets_arr, k, gc_lo, gc_hi)
            lap("fin_props")
            dimer = self._self_dimer(sets_list)                               # core:487-503 for all windows at once
            lap("fin_dimer")
        else:
            # primer properties and the self-dimer test depend on the primer only: every rank takes every world-th primer
            # and the values are shared (one small collective; float values travel as bit patterns)
            sel = np.arange(rank, n, world)
            part = np.zeros((n, 6), np.int64)
            if len(sel):
                p_tm, p_gc, p_fl, p_deg, p_ndeg = self._primer_props(sets_arr[sel], k, gc_lo, gc_hi)
                lap("fin_props")
                p_dim = self._self_dimer([sets_list[i] for i in sel.tolist()])
                part[sel, 0] = np.asarray(p_tm, np.float64).view(np.int64)
                part[sel, 1] = np.asarray(p_gc, np.float64).view(np.int64)
                part[sel, 2], part[sel, 3], part[sel, 4] = p_fl, p_deg, p_ndeg
                part[sel, 5] = np.asarray(p_dim, np.int64)
            lap("fin_dimer")
            part = self.comm.allreduce_sum(part)
            tm_avg, gc = part[:, 0].copy().view(np.float64), part[:, 1].copy().view(np.float64)
            flags, deg, ndeg, dimer = part[:, 2], part[:, 3], part[:, 4], part[:, 5]
            lap("fin_share")
        if self.rows_on_rank0_only and rank != 0 and not self.sidecars:
            return []                  # rows are identical on every rank: only rank 0 assembles (and writes) them
        seqkeys = self.msa.seqkeys(k, pos) if self.sidecars else None
        lut = np.frombuffer(CODE_CHARS.encode(), dtype=np.uint8)
        trace_str = None
        if res["trace"] is not None:
            trace_str = lut[res["trace"][:int(res["trace_off"][n]), :k]].view("S%d" % k).ravel().astype(str).tolist()
        # core:846: expansions that are not keys of `cover`; the defaultdict look-ups of the seeds (core:787-835) added
        # their strings as keys, observed or not: a seed nobody carries that the final primer matches is one key more
        seeds = np.asarray(res["seeds"])[:, :, :k]
        matched = ((sets_arr[:, None, :k] >> seeds) & 1).all(axis=2)                     # [window, track]
        live = np.arange(2)[None, :] < np.asarray(res["ntracks"])[:, None]
        ghost = (matched & live & (np.asarray(res["seed_cover"]) == 0)).sum(axis=1)
        nonsense_all = (np.asarray(deg, np.int64) - np.asarray(distinct, np.int64) - ghost).tolist()
        strings = lut[sets_arr[:, :k]].view("S%d" % k).ravel().astype(str).tolist()     # primer_string() of every row
        out = []
        for i in range(n):
            wi, p, c_bit, t_bit, cover_number, _ = keep[i]
            sets = sets_list[i]
            nonsense = nonsense_all[i]
            if dimer[i]:
                continue                                                  # core:749-751
            fl = int(flags[i])
            notes = []
            if fl & 1:
                notes.append("GC_out_of_range (" + str(float(gc[i])) + ")")
            if fl & 2:
                notes.append("di_nucleotide")
            if fl & 4:
                notes.append("hairpin")
            init, fm, rm = (int(x) for x in res["counts"][i, :3])
            row = [p, c_bit, t_bit, strings[i], int(ndeg[i]), nonsense, int(perfect[i]), init + fm,
                   init + rm, float(tm_avg[i]), float(gc[i]) if not notes else "|".join(notes)]
            rec = {"row": row}
            if trace_str is not None:
                a, b = int(res["trace_off"][i]), int(res["trace_off"][i + 1])
                rec["trace"] = trace_str[a:b]
            if self.sidecars:
                rec["non_cov"], rec["gap_ids"] = self._sidecars(hist, wi, p, sets, bits[i], seqkeys[i])
            out.append(rec)
        self.stats["accepted"] += len(out)
        lap("fin_rows")
        return out

    def _primer_props(self, sets_arr, k, gc_lo, gc_hi):
        """Tm average, GC content and filter flags of the chosen primers (core:849-852, 507-521)"""
        if not hasattr(self.ctx, "h"):                 # injected test backend
            return self.ctx.primer_props(sets_arr, k, gc_lo, gc_hi, self.distance, TM_CONSTS)
        tm_avg, gc, flags, deg, ndeg = self.ctx.primer_props(sets_arr, k, gc_lo, gc_hi, self.distance, TM_CONSTS)
        for i in np.nonzero(flags & (64 | 128))[0].tolist():      # a mean on a rounding tie: exact rational replay
            sets = sets_arr[i, :k].tolist()
            if flags[i] & 64:
                raw = self.ctx.tm(expand_array(sets), TM_CONSTS)
                tm_avg[i] = round(exact_mean([round(float(x), 2) for x in raw]), 2)
            if flags[i] & 128:
                gc[i] = gc_content(sets)
                flags[i] = (flags[i] & ~1) | (0 if gc_lo <= gc[i] <= gc_hi else 1)
        return tm_avg, gc, flags, deg, ndeg

    def _sidecars(self, hist, wi, pos, sets, bits, keys):
        """core:1116-1125 / 696-698: {haplotype: [ids]} of the sequences the final primer does not cover (F, R) and
        of the gap rows, rebuilt from the scan's per-sequence bits and the per-sequence table keys"""
        k, v = self.primer_length, self.variation
        N = self.n_local
        ids = self.ids
        unpack = lambda words: np.unpackbits(words.view(np.uint8), bitorder="little")[:N].astype(bool)
        non_f, non_r, gap = unpack(bits[0]), unpack(bits[1]), unpack(bits[2])
        iupac = keys == np.uint64(_lib.KEY_IUPAC)
        groups = ({}, {}, {})                      # F non-cover, R non-cover, gap rows: haplotype -> [sequence index]
        for flag, dct in zip((non_f, non_r, gap), groups):
            by_key = {}
            for s in np.nonzero(flag & ~iupac)[0].tolist():       # plain rows: one haplotype per sequence
                by_key.setdefault(int(keys[s]), []).append(s)
            for key, ss in by_key.items():
                dct[_key_string(key, k)] = ss
        # rows whose window holds IUPAC cells: every expansion is its own haplotype (rare; replayed on the host copy)
        for s in np.nonzero(iupac)[0].tolist():
            wsets = list(self._window_cells(s, pos))
            is_gap = sum(1 for c in wsets if c == 0) > v
            for hap in expand_strings(wsets):
                if is_gap:
                    groups[2].setdefault(hap, []).append(s)
                    continue
                m = 0
                for i, ch in enumerate(hap):
                    if ch == "-" or not (sets[i] >> BASES.index(ch)) & 1:
                        m |= 1 << i
                if not m:
                    continue
                far = bin(m).count("1") > v
                if far or m & self.fmask:
                    groups[0].setdefault(hap, []).append(s)
                if far or m & self.rmask:
                    groups[1].setdefault(hap, []).append(s)
        f_dict, r_dict, g_dict = ({hap: [ids[s] for s in sorted(ss)] for hap, ss in dct.items()} for dct in groups)
        return [f_dict, r_dict], g_dict

    def _self_dimer(self, sets_list):
        if hasattr(self.ctx, "h"):
            from .dimer import dimer_flags
            return dimer_flags(self.ctx, sets_list)
        return self.ctx.dimer_flags(sets_list)       # injected test backend

    # -- core:1133-1180 -------------------------------------------------------------------------------------
    def run(self):
        """core:1133-1180: the .out TSV and the side files.  The reference's JSON side files list sequence ids per
        uncovered haplotype and window — megabytes at 500 sequences, unusable at 10^6 — so above SIDE_JSON_MAX sequences
        (or with sidecar_format="bits") the same information is written as per-sequence bit vectors instead
        (<out>.coverage_bits.npz: F non-cover / R non-cover / gap row per chosen primer), which is what the pairing
        step (pairing.py) actually consumes (SURVEY.md 8f-1).  Below the threshold the files are the reference's."""
        k = self.primer_length
        fmt = self.sidecar_format
        if fmt == "auto":
            fmt = "json" if self.total_sequence_number <= SIDE_JSON_MAX else "bits"
        want_json = self.sidecars and fmt == "json"
        want_bits = self.sidecars and fmt == "bits"
        saved = (self.sidecars, self.keep_bits)
        self.sidecars, self.keep_bits = want_json, want_bits or self.keep_bits
        try:
            recs = self.design(range(self.start_position, self.stop_position - k))
        finally:
            self.sidecars, self.keep_bits = saved[0], saved[1]
        recs.sort(key=lambda r: r["row"][0])
        if self.comm.rank == 0:
            with open(self.outfile, "w") as fo:
                fo.write("\t".join(TSV_HEADER) + "\n")
                for r in recs:
                    fo.write("\t".join(map(str, r["row"])) + "\n")
        if want_bits:
            self.write_bits(self.outfile)
        if not want_json:
            return recs
        non_cov = {r["row"][0]: r["non_cov"] for r in recs}
        gap_ids = {r["row"][0]: r["gap_ids"] for r in recs}
        if self.comm.world > 1:                 # shards hold disjoint id lists: concatenate them in rank order
            non_cov, gap_ids = _merge_sidecars(self.comm.allgather_object((non_cov, gap_ids)))
            if self.comm.rank != 0:
                return recs
        with open(self.outfile + ".non_coverage_seq_id_json", "w") as fj:
            json.dump(non_cov, fj, indent=4)
        with open(self.outfile + ".gap_seq_id_json", "w") as fg:
            json.dump(gap_ids, fg, indent=4)
        return recs

    def coverage_bits(self):
        """(positions int32[n], bits uint32[n, 3, words]) of the last design(): F non-cover, R non-cover and gap-row
        bit vectors of every chosen primer over this process's sequences (host copy)"""
        pos, bits = [], []
        for p, b in self.bit_vectors:
            pos.append(np.asarray(p, np.int32))
            bits.append(b.to_host() if hasattr(b, "to_host") else np.asarray(b))
        words = (self.n_local + 31) // 32
        if not pos:
            return np.zeros(0, np.int32), np.zeros((0, 3, words), np.uint32)
        return np.concatenate(pos), np.concatenate(bits)[:, :, :words]

    def write_bits(self, out: str):
        """<out>.coverage_bits.npz (one per rank in a sequence-sharded run: shards hold disjoint sequences)"""
        pos, bits = self.coverage_bits()
        np.savez(bits_file(out, self.comm.rank, self.comm.world), positions=pos, bits=bits, n_local=self.n_local,
                 row0=self.row0, n_total=self.total_sequence_number, world=self.comm.world)

    def close(self):
        self.msa.close()
        self.ctx.close()


# ----------------------------------------------------------------------------------------------------------
def _merge_sidecars(parts):
    non_cov, gap_ids = {}, {}
    for nc, gi in parts:
        for pos, (f, r) in nc.items():
            tgt = non_cov.setdefault(pos, [{}, {}])
            for src, dst in ((f, tgt[0]), (r, tgt[1])):
                for hap, ids in src.items():
                    dst.setdefault(hap, []).extend(ids)
        for pos, d in gi.items():
            tgt = gap_ids.setdefault(pos, {})
            for hap, ids in d.items():
                tgt.setdefault(hap, []).extend(ids)
    return non_cov, gap_ids


SIDE_JSON_MAX = 20000      # sequences up to which run() writes the reference's JSON side files


def bits_file(out: str, rank: int = 0, world: int = 1) -> str:
    return out + (".coverage_bits.npz" if world == 1 else ".coverage_bits.%dof%d.npz" % (rank, world))


class _AllMerged:
    def __getitem__(self, i):
        return True


ALL_MERGED = _AllMerged()


def exact_mean(vals) -> float:
    """statistics.mean of floats (exact rational mean, correctly rounded once) without Fractions: every value is
    scaled by 2^60 exactly (holds for 2^-8 <= |x| < 2^11, i.e. any Tm / GC fraction; else fall back)"""
    arr = np.asarray(vals, np.float64)
    mag = np.abs(arr)
    if len(arr) and bool(((mag >= 1.0) & (mag < 1024.0)).all()):
        # 1 <= |x| < 2^10: a multiple of 2^-52 below 2^10, so x * 2^52 is an integer below 2^62 (exact in int64)
        return sum((arr * 4503599627370496.0).astype(np.int64).tolist()) / (len(arr) << 52)
    if all((x == 0.0) or (0.00390625 <= abs(x) < 2048.0) for x in vals):
        total = 0
        for x in vals:
            total += int(x * 1152921504606846976.0)
        return total / (len(vals) << 60)
    return mean(vals)


def _default_batch(n_seq: int) -> int:
    # table bytes per window = 20 * 2^ceil(log2(2n+64)); keep a batch under ~32 GB of the 80 GB HBM
    cap = 1 << max(6, int(math.ceil(math.log2(2 * n_seq + 64))))
    return max(1, min(4096, int(32e9 // (20 * cap))))


def _near_half(x: float) -> bool:
    """x*100 within 1e-6 of a rounding boundary"""
    y = x * 100.0
    return abs((y - math.floor(y)) - 0.5) < 1e-6


def _count_gap_digits(x: int, k: int) -> int:
    n = 0
    for _ in range(k):
        n += (x % 5) == 4
        x //= 5
    return n


def _key_bases(key: int, k: int):
    """gap-free table key -> base indices"""
    mask = (1 << k) - 1
    b0, b1 = key & mask, (key >> k) & mask
    return [((b0 >> i) & 1) | (((b1 >> i) & 1) << 1) for i in range(k)]


def _key_string(key: int, k: int) -> str:
    if key < _lib.KEY_BASE5:
        return "".join(BASES[b] for b in _key_bases(key, k))
    x = key - _lib.KEY_BASE5
    out = []
    for _ in range(k):
        out.append("ACGT-"[x % 5])
        x //= 5
    return "".join(out)


def main(argv=None):
    from .cli_core import main as cli_main
    return cli_main(argv)
