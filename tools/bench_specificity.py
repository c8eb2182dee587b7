#!/usr/bin/env python
"""All-combinations in-silico PCR benchmark (primer_specificity.py; DESIGN.md §4, profiles/h100_bench_specificity.json);
prints one JSON line.

    python tools/bench_specificity.py --steps 3 --warmup 1 [--targets 65536]

Workload: the panel of tools/bench_pcr.py — 48 primer pairs (96 primers, 9 216 combinations), v = 3, -c 1,2,-1,
products of 50..2000 bases, against a seeded synthetic database of about 65 536 targets of about 10 kb
(multiprime_b200/synth.py write_pcr_targets), written to a temporary directory.  The panel tiles one genome, so most of
its products are cross-pair products.  The card's name, SM clock and enforced power limit are recorded the way bench.py
records them for the scan."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler  # noqa: E402

KERNELS = ("k_pattern_sites", "k_products_filter", "k_products_sort", "k_products_segments", "k_products_join",
           "k_products_reduce", "k_products_summary")


def run_specificity(args):
    """call = mpb_pattern_products with the targets resident in HBM (search, filter, sorts, join, merge, summary and the
    copy-back of the summaries and listed rows); e2e = the whole tool from the FASTA file to its two output files"""
    import shutil
    import tempfile
    import torch
    from multiprime_b200 import _lib, synth
    from multiprime_b200 import primer_coverage as pc
    from multiprime_b200 import primer_specificity as ps
    tmp = tempfile.mkdtemp(prefix="mpb_spec_")
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
        primers = ps.Primers(panel)
        rows, width, starts = pc.layout(targets, panel.lmax)
        msa = _lib.Msa(ctx, rows, len(rows), width, row_bytes=rows.shape[1])
        n = len(primers.seqs)

        def call():
            return msa.pattern_products(panel.allow, panel.plen, panel.strict, v, primers.pat_primer, primers.pat_side,
                                        n, pc.S, starts, targets.lens, size[0], size[1], primers.listed, ps.MAX_ROWS)

        for _ in range(args.warmup):
            res = call()
        sampler = ClockSampler(0)
        sampler.start()
        ctx.profile_read(None)
        ctx.profile(True)
        call_ms = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            res = call()
            call_ms.append(1000 * (time.perf_counter() - t0))
        kernels = {}
        for k in KERNELS:
            ms, launches, _ = ctx.profile_read(k)
            kernels[k + "_ms"] = ms / args.steps
            kernels[k + "_launches"] = launches // args.steps
        ctx.profile(False)
        sampler.stop_flag.set()
        msa.close()
        e2e_s = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            ps.run(fa, pairs, os.path.join(tmp, "out"), v, coord, size)
            e2e_s.append(time.perf_counter() - t0)
        comb = res["comb"]
        call_med = statistics.median(call_ms)
        print(json.dumps({
            "metric": "products_per_sec", "value": int(comb[:, :, 0].sum()) / (call_med / 1000), "unit": "products/s",
            "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "higher_is_better": True, "data": "synthetic",
            "config": {"workload": "all-combinations in-silico PCR, %d pairs (%d primers) v=%d -c %s -s %d,%d against "
                                   "%d synthetic targets (%d bases, seed 20241015)"
                                   % (len(pairs), n, v, coord, size[0], size[1], len(targets.names),
                                      int(targets.lens.sum())),
                       "rows": len(rows), "row_width": width, "generate_s": round(gen_s, 2)},
            "counts": {"search_hits": int(res["stats"][0]), "left_sites": int(res["stats"][1]),
                       "right_sites": int(res["stats"][2]), "products": int(comb[:, :, 0].sum()),
                       "products_unintended": int(comb[:, :, 0][primers.klass != 0].sum()),
                       "groups": int(res["stats"][3]), "listed_rows": int(res["n_listed"]),
                       "unintended_targets": int(res["union"][0])},
            "call_ms_min_median_max": [round(min(call_ms), 2), round(call_med, 2), round(max(call_ms), 2)],
            "kernels": kernels,
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
    run_specificity(ap.parse_args())
