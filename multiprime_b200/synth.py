"""Deterministic synthetic MSA generator (the "10^6 x 600" north-star workload and its small siblings).

Mutation model after SURVEY.md section 8(d) "C4 synthetic" (conserved / variable 60-column blocks,
8 clades, terminal and internal gap runs, sparse 2-fold IUPAC cells), but drawn in fixed row chunks
of CHUNK rows, each chunk from its own PCG64 stream keyed by (seed, chunk index), so that any row
range can be produced without generating the rows before it (needed to shard 10^6 rows over ranks).

Cells are returned as 4-bit base sets: A=1, C=2, G=4, T=8, IUPAC = OR of its bases, gap = 0.
"""
from __future__ import annotations

import numpy as np

CHUNK = 8192
CODE_CHARS = "-ACMGRSVTWYHKDBN"          # index = 4-bit set (A=1,C=2,G=4,T=8)
_CLADE_P = [.40, .20, .12, .10, .08, .05, .03, .02]
# 2-fold codes containing base b (A,C,G,T): A->R,M,W  C->Y,M,S  G->R,K,S  T->Y,K,W
_TWOFOLD = np.array([[1 | 4, 1 | 2, 1 | 8], [2 | 8, 1 | 2, 2 | 4], [1 | 4, 4 | 8, 2 | 4], [2 | 8, 4 | 8, 1 | 8]],
                    dtype=np.uint8)


def _plan(seed: int, n_col: int):
    rng = np.random.Generator(np.random.PCG64([seed, 0xC4]))
    root = rng.integers(0, 4, n_col)
    mu = np.where((np.arange(n_col) // 60) % 2 == 0, 0.01, 0.12)
    cols = np.stack([rng.choice(n_col, 6, replace=False) for _ in range(8)])
    subs = np.stack([rng.integers(1, 4, 6) for _ in range(8)])
    return root, mu, cols, subs


def synth_codes(n_seq: int, n_col: int = 600, seed: int = 20240923, row0: int = 0,
                gap_rate: float = 0.002, iupac_rate: float = 1e-4, term_gap: float = 0.05) -> np.ndarray:
    """rows [row0, row0+n_seq) of the synthetic alignment as uint8 4-bit sets, shape (n_seq, n_col)"""
    root, mu, ccols, csubs = _plan(seed, n_col)
    out = np.empty((n_seq, n_col), dtype=np.uint8)
    r = row0
    while r < row0 + n_seq:
        c = r // CHUNK
        lo, hi = c * CHUNK, (c + 1) * CHUNK
        block = _chunk(seed, c, n_col, root, mu, ccols, csubs, gap_rate, iupac_rate, term_gap)
        a, b = max(r, lo), min(row0 + n_seq, hi)
        out[a - row0:b - row0] = block[a - lo:b - lo]
        r = b
    return out


def _chunk(seed, c, n_col, root, mu, ccols, csubs, gap_rate, iupac_rate, term_gap):
    rng = np.random.Generator(np.random.PCG64([seed, 1, c]))
    n = CHUNK
    clade = rng.choice(8, n, p=_CLADE_P)
    x = np.broadcast_to(root.astype(np.uint8), (n, n_col)).copy()
    for k in range(8):
        rows = np.nonzero(clade == k)[0]
        x[np.ix_(rows, ccols[k])] = ((root[ccols[k]] + csubs[k]) % 4).astype(np.uint8)
    mut = rng.random((n, n_col), dtype=np.float32) < mu.astype(np.float32)
    shift = rng.integers(1, 4, (n, n_col), dtype=np.uint8)
    x = np.where(mut, (x + shift) % 4, x).astype(np.uint8)
    code = (np.uint8(1) << x).astype(np.uint8)
    # terminal gap runs
    lead = rng.random(n) < term_gap
    trail = rng.random(n) < term_gap
    lead_len = rng.integers(1, 31, n)
    trail_len = rng.integers(1, 31, n)
    col = np.arange(n_col)
    code[(col[None, :] < (lead_len * lead)[:, None])] = 0
    code[(col[None, :] >= (n_col - trail_len * trail)[:, None])] = 0
    # internal gap runs, geometric length with mean 3
    starts = np.argwhere(rng.random((n, n_col), dtype=np.float32) < np.float32(gap_rate / 3))
    glen = rng.geometric(1 / 3, len(starts))
    for d in range(int(glen.max()) if len(glen) else 0):
        sel = (glen > d) & (starts[:, 1] + d < n_col)
        code[starts[sel, 0], starts[sel, 1] + d] = 0
    # sparse 2-fold IUPAC cells
    amb = np.argwhere((rng.random((n, n_col), dtype=np.float32) < np.float32(iupac_rate)) & (code != 0))
    pick = rng.integers(0, 3, len(amb))
    base = x[amb[:, 0], amb[:, 1]]
    code[amb[:, 0], amb[:, 1]] = _TWOFOLD[base, pick]
    return code


def synth_codes_parallel(n_seq: int, n_col: int = 600, seed: int = 20240923, row0: int = 0, procs: int = 0,
                         **kw) -> np.ndarray:
    """synth_codes() with the chunks drawn by a process pool (same result, chunk streams are independent)"""
    import os
    from concurrent.futures import ProcessPoolExecutor
    procs = procs or min(32, os.cpu_count() or 1)
    bounds = list(range(row0 - row0 % CHUNK, row0 + n_seq, CHUNK))
    jobs = [(max(b, row0), min(b + CHUNK, row0 + n_seq)) for b in bounds]
    if procs <= 1 or len(jobs) <= 1:
        return synth_codes(n_seq, n_col, seed, row0, **kw)
    out = np.empty((n_seq, n_col), dtype=np.uint8)
    # (forks: call this before CUDA / NCCL threads exist in the process, as bench.py does)
    with ProcessPoolExecutor(procs) as ex:
        futs = [(a, b, ex.submit(synth_codes, b - a, n_col, seed, a, **kw)) for a, b in jobs]
        for a, b, f in futs:
            out[a - row0:b - row0] = f.result()
    return out


def codes_to_strings(codes: np.ndarray) -> list[str]:
    lut = np.frombuffer(CODE_CHARS.encode(), dtype=np.uint8)
    return [row.tobytes().decode() for row in lut[codes]]


def seq_ids(n_seq: int, row0: int = 0) -> list[str]:
    return [">s%07d" % (row0 + i) for i in range(n_seq)]


def write_fasta(path: str, codes: np.ndarray, row0: int = 0) -> None:
    with open(path, "w") as fh:
        for sid, s in zip(seq_ids(len(codes), row0), codes_to_strings(codes)):
            fh.write(sid + "\n" + s + "\n")


_COMP = np.array([3, 2, 1, 0], np.uint8)          # base index (A,C,G,T) -> complement


def write_pcr_targets(path: str, n_targets: int = 65536, length: int = 10_000, n_pairs: int = 48, seed: int = 20241015):
    """The in-silico PCR workload (tools/bench_pcr.py): a FASTA of n_targets unaligned targets of about `length`
    bases from a clade-structured root — 8 clades with their own substitutions, 1 % point mutations, a few short indels,
    random trims of up to 200 bases at each end, half of the targets reverse-complemented — and n_pairs primer pairs
    (20-mers) cut from the root, a third of them with one or two degenerate positions.  Returns {name: (F, R)}."""
    rng = np.random.Generator(np.random.PCG64([seed, 0x9C2]))
    root = rng.integers(0, 4, length).astype(np.uint8)
    clade_cols = rng.choice(length, (8, 40))
    clade_shift = rng.integers(1, 4, (8, 40)).astype(np.uint8)
    letters = np.frombuffer(b"ACGT", np.uint8)
    pairs = {}
    starts = np.sort(rng.choice(np.arange(100, length - 1700), n_pairs, replace=False))
    for q, a in enumerate(starts.tolist()):
        b = a + int(rng.integers(200, 1500))
        f = ["ACGT"[x] for x in root[a:a + 20]]
        r = ["ACGT"[3 - x] for x in root[b:b + 20][::-1]]
        if q % 3 == 0:
            for p in rng.choice(np.arange(3, 17), int(rng.integers(1, 3)), replace=False):
                f[p] = {"A": "R", "G": "R", "C": "Y", "T": "Y"}[f[p]]
        pairs["pair%02d" % q] = ("".join(f), "".join(r))
    chunk = 4096
    with open(path, "wb") as fh:
        for c0 in range(0, n_targets, chunk):
            n = min(chunk, n_targets - c0)
            x = np.broadcast_to(root, (n, length)).copy()
            clade = rng.integers(0, 8, n)
            for k in range(8):
                rows = np.nonzero(clade == k)[0]
                x[np.ix_(rows, clade_cols[k])] = (x[np.ix_(rows, clade_cols[k])] + clade_shift[k]) % 4
            mut = rng.random((n, length), dtype=np.float32) < 0.01
            x = np.where(mut, (x + rng.integers(1, 4, (n, length), dtype=np.uint8)) % 4, x).astype(np.uint8)
            out = []
            for i in range(n):
                s = x[i]
                for _ in range(int(rng.poisson(2))):
                    p, d = int(rng.integers(0, len(s) - 8)), int(rng.integers(1, 6))
                    s = np.delete(s, np.arange(p, p + d)) if rng.random() < 0.5 else \
                        np.insert(s, p, rng.integers(0, 4, d).astype(np.uint8))
                s = s[int(rng.integers(0, 200)):len(s) - int(rng.integers(0, 200))]
                if (c0 + i) % 2:
                    s = _COMP[s[::-1]]
                out.append(b">t%07d\n" % (c0 + i) + letters[s].tobytes() + b"\n")
            fh.write(b"".join(out))
    return pairs


def pcr_candidate_pool(n_pairs: int = 2048, length: int = 10_000, seed: int = 20241015):
    """A candidate pool for the targets of write_pcr_targets (tools/bench_select.py): the generator's first draws (root,
    clade columns, clade shifts) are replayed, and 20-mer pairs (products of 220..1320 bases) are cut in turn from the
    root and from its 8 clade variants.  Most forward primers end on a clade column, whose base is then a strict 3'
    mismatch on the targets of some clades, so no single pair amplifies every target.  write_pcr_targets' output does
    not depend on this function.  Returns {name: (F, R)}."""
    rng = np.random.Generator(np.random.PCG64([seed, 0x9C2]))
    root = rng.integers(0, 4, length).astype(np.uint8)
    clade_cols = rng.choice(length, (8, 40))
    clade_shift = rng.integers(1, 4, (8, 40)).astype(np.uint8)
    variants = [root]
    for k in range(8):
        x = root.copy()
        x[clade_cols[k]] = (x[clade_cols[k]] + clade_shift[k]) % 4
        variants.append(x)
    pick = np.random.Generator(np.random.PCG64([seed, 0x5E1]))
    pairs = {}
    for q in range(n_pairs):
        src = variants[q % 9]
        a = int(clade_cols[int(pick.integers(0, 8)), int(pick.integers(0, 40))]) - 19
        if not 250 <= a <= length - 1600 or pick.random() < 0.2:
            a = int(pick.integers(250, length - 1600))
        b = a + int(pick.integers(200, 1300))
        f = "".join("ACGT"[x] for x in src[a:a + 20])
        r = "".join("ACGT"[3 - x] for x in src[b:b + 20][::-1])
        pairs["cand%04d_v%d" % (q, q % 9)] = (f, r)
    return pairs


def write_pcr_background(path: str, n_random: int = 256, random_length: int = 10_000, n_copies: int = 4,
                         copy_span=(0, 3000), divergence: float = 0.02, length: int = 10_000, seed: int = 20241015):
    """A background for primer_select --background (tools/bench_select_specific.py): n_random records of uniform random
    bases, which no 20-mer of the pool binds with a few mismatches by chance, and n_copies copies of root[copy_span]
    of write_pcr_targets (the generator's first draw, replayed) with `divergence` point substitutions each, so the
    candidates of pcr_candidate_pool whose sites both fall in copy_span have products there (off-target) and the
    others do not.  Returns the number of records."""
    rng = np.random.Generator(np.random.PCG64([seed, 0x9C2]))
    root = rng.integers(0, 4, length).astype(np.uint8)
    bg = np.random.Generator(np.random.PCG64([seed, 0xB6]))
    with open(path, "w") as fh:
        for k in range(n_random):
            fh.write(">random%05d\n%s\n" % (k, "".join("ACGT"[x] for x in bg.integers(0, 4, random_length))))
        for k in range(n_copies):
            x = root[copy_span[0]:copy_span[1]].copy()
            hit = bg.random(len(x)) < divergence
            x[hit] = (x[hit] + bg.integers(1, 4, int(hit.sum()))) % 4
            fh.write(">root_copy%d\n%s\n" % (k, "".join("ACGT"[c] for c in x)))
    return n_random + n_copies
