#!/usr/bin/env python
"""In-silico PCR benchmark (primer_coverage.py; DESIGN.md §4, profiles/h100_bench_pcr.json); prints one JSON line.

    python tools/bench_pcr.py --steps 3 --warmup 1 [--targets 65536]

Workload: 48 primer pairs, v = 3, -c 1,2,-1, products of 50..2000 bases, against a seeded synthetic database of about
65 536 targets of about 10 kb (multiprime_b200/synth.py write_pcr_targets), written to a temporary directory.  The card's
name, SM clock and enforced power limit are recorded the way bench.py records them for the scan."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler  # noqa: E402


def run_pcr(args):
    """in-silico PCR (primer_coverage.py): 48 primer pairs, v = 3, -c 1,2,-1, products of 50..2000 bases, against a
    seeded synthetic database of about 65 536 targets of about 10 kb (multiprime_b200/synth.py write_pcr_targets), written
    to a temporary directory.  value = pattern x position x sequence evaluations of mpb_pattern_sites per second with the
    targets resident in HBM (call time: kernel, site copy-back and sort); e2e = the whole tool from the FASTA file to its
    two output files.  k_pattern_hits on the same rows and patterns (exact matching) is timed for comparison."""
    import shutil
    import tempfile
    import numpy as np
    import torch
    from multiprime_b200 import _lib, synth
    from multiprime_b200 import primer_coverage as pc
    tmp = tempfile.mkdtemp(prefix="mpb_pcr_")
    try:
        fa = os.path.join(tmp, "targets.fa")
        t0 = time.perf_counter()
        pairs = synth.write_pcr_targets(fa, args.targets)
        gen_s = time.perf_counter() - t0
        v, coord, size = 3, "1,2,-1", (50, 2000)
        torch.cuda.set_device(0)
        ctx = _lib.Context.shared(0)
        targets = pc.read_targets(fa)
        panel = pc.Panel(pairs, coord)
        rows, width, starts = pc.layout(targets, panel.lmax)
        msa = _lib.Msa(ctx, rows, len(rows), width, row_bytes=rows.shape[1])

        def search():
            return msa.pattern_sites(panel.allow, panel.plen, panel.strict, v, max_hits=1 << 24)

        for _ in range(args.warmup):
            hp, hr, hx, hm = search()
        sampler = ClockSampler(0)
        sampler.start()
        ctx.profile_read(None)
        ctx.profile(True)
        call_ms = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            hp, hr, hx, hm = search()
            call_ms.append(1000 * (time.perf_counter() - t0))
        k_ms, k_n, units = ctx.profile_read("k_pattern_sites")
        for _ in range(args.steps):
            msa.pattern_hits(panel.allow, panel.plen, max_hits=1 << 24)
        x_ms, x_n, _ = ctx.profile_read("k_pattern_hits")
        ctx.profile(False)
        sampler.stop_flag.set()
        msa.close()
        pair_ms = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            sites = pc.stream_sites(*(np.asarray(a, np.int64) for a in (hp, hr, hx, hm)), panel.plen.astype(np.int64),
                                    starts, targets.lens)
            best = pc.amplicons(sites, panel, targets.lens, size[0], size[1], v)
            pair_ms.append(1000 * (time.perf_counter() - t0))
        e2e_s = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            pc.run(fa, pairs, os.path.join(tmp, "out"), v, coord, size)
            e2e_s.append(time.perf_counter() - t0)
        evals = units / max(1, k_n)
        amplified = len(set().union(*(b["rec"].tolist() for b in best)))
        print(json.dumps({
            "metric": "pattern_x_position_x_sequence_evals_per_sec", "value": evals / (statistics.median(call_ms) / 1000),
            "unit": "evals/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "higher_is_better": True,
            "data": "synthetic",
            "config": {"workload": "in-silico PCR, %d pairs (%d patterns) v=%d -c %s -s %d,%d against %d synthetic targets "
                                   "(%d bases, seed 20241015)" % (len(pairs), len(panel.plen), v, coord, size[0], size[1],
                                                                  len(targets.names), int(targets.lens.sum())),
                       "rows": len(rows), "row_width": width, "evals_per_call": evals, "sites": len(hp),
                       "amplified_targets_any_pair": amplified, "generate_s": round(gen_s, 2)},
            "search_call_ms_min_median_max": [round(min(call_ms), 2), round(statistics.median(call_ms), 2),
                                              round(max(call_ms), 2)],
            "kernels": {"k_pattern_sites_ms": k_ms / max(1, k_n), "k_pattern_hits_ms_same_patterns_exact": x_ms / max(1, x_n),
                        "kernel_evals_per_sec": evals / (k_ms / max(1, k_n) / 1000)},
            "host_pairing_ms": statistics.median(pair_ms),
            "e2e_s_from_fasta": statistics.median(e2e_s),
            "device": torch.cuda.get_device_name(0),
            "clocks": sampler.summary()}))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--targets", type=int, default=65536, help="synthetic targets")
    run_pcr(ap.parse_args())
