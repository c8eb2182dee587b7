#!/usr/bin/env python
"""primer_select --cross / --background benchmark (DESIGN.md §4, profiles/h100_bench_select_specific.json); prints one
JSON line.

    python tools/bench_select_specific.py --steps 2 --warmup 1 [--targets 65536] [--pairs 2048]

Workload: tools/bench_select.py's (the targets of synth.write_pcr_targets, a pool of synth.pcr_candidate_pool, v = 3,
-c 1,2,-1, -s 50,2000) plus the background of synth.write_pcr_background: random records and diverged copies of the
first 3 kb of the root, so the candidates with both sites there go off-target.  The pool tiles one genome, so --cross
excludes most candidates after the first take: the densest join.
build    the matrix build without and with keeping the sites (alternated, the same blocks), the seal sort, the list's
         sites and its device bytes;
cross    k_sites_pick / k_sites_cross ms per taken pair in a tool run with --cross;
own      the background list's build (wall) and the own join (re-key sort and k_sites_own, CUDA events);
tool     the whole tool from the FASTA files to its three outputs: no flag, --cross, --background, both; steps taken and
         the candidates of each status.
The card's name, SM clock and enforced power limit are recorded the way bench.py records them."""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler  # noqa: E402

V, SIZE = 3, (50, 2000)


def run_build(ctx, targets, pairs, steps, warmup):
    import numpy as np
    from multiprime_b200 import _lib
    from multiprime_b200 import primer_select as sel
    pool = sel.Pool(pairs, {}, "1,2,-1")
    block = sel.block_of(len(targets.names), len(pool.names))
    walls = {False: [], True: []}
    n_sites = 0
    for it in range(warmup + steps):
        for keep in (False, True):
            if it == warmup + steps - 1 and keep:
                ctx.profile_read(None)
                ctx.profile(True)
            t0 = time.perf_counter()
            built = sel.build_matrix(targets, pool.panel, V, SIZE[0], SIZE[1], 0, None, _lib, block,
                                     np.zeros(3, np.int64), keep_sites=keep)
            ctx.sync()
            if it >= warmup:
                walls[keep].append(time.perf_counter() - t0)
            built[1].close()
            if keep:
                n_sites = len(built[2].keys()) if it == warmup + steps - 1 else n_sites
                built[2].close()
    seal_ms, _, _ = ctx.profile_read("k_sites_seal")
    keep_ms, keep_n, _ = ctx.profile_read("k_sites_keep")
    ctx.profile(False)
    return {"pairs": len(pairs), "targets": len(targets.names), "block_pairs": block,
            "build_s_without_sites": [round(w, 3) for w in walls[False]],
            "build_s_keeping_sites": [round(w, 3) for w in walls[True]],
            "keep_append_ms_total": round(keep_ms, 2), "keep_calls": keep_n, "seal_sort_ms": round(seal_ms, 2),
            "sites": n_sites, "site_list_bytes": 8 * n_sites}


def run_tool(ctx, fa, bgfa, pairs, steps, warmup, flags):
    from multiprime_b200 import primer_select as sel
    tmp = tempfile.mkdtemp(prefix="mpb_select_specific_out_")
    try:
        e2e, times = [], {}
        for it in range(warmup + steps):
            if it == warmup + steps - 1:
                ctx.profile_read(None)
                ctx.profile(True)
            times = {}
            t0 = time.perf_counter()
            res = sel.run(fa, pairs, os.path.join(tmp, "o"), V, "1,2,-1", SIZE, cross=flags.get("cross", False),
                          background=bgfa if flags.get("background") else None, _times=times)
            if it >= warmup:
                e2e.append(time.perf_counter() - t0)
        prof = {n: ctx.profile_read(n) for n in ("k_sites_pick", "k_sites_cross", "k_sites_own_sort", "k_sites_own")}
        ctx.profile(False)
        status = {}
        with open(os.path.join(tmp, "o.candidates.tsv")) as fh:
            for line in fh.read().splitlines()[1:]:
                s = line.split("\t")[5]
                status[s] = status.get(s, 0) + 1
        out = {"flags": sorted(k for k, v in flags.items() if v), "steps_taken": times["steps"],
               "covered": res["covered"], "total": res["total"], "status": status,
               "read_s": round(times["read"], 3), "cover_s": round(times["cover"], 3),
               "background_s": round(times["background"], 3), "dimer_s": round(times["dimer"], 3),
               "greedy_s": round(times["greedy"], 3), "e2e_s": [round(x, 3) for x in e2e],
               "e2e_s_median": round(statistics.median(e2e), 3)}
        pick_ms, pick_n, _ = prof["k_sites_pick"]
        cross_ms, cross_n, _ = prof["k_sites_cross"]
        if cross_n:
            out.update(cross_calls=cross_n, pick_ms_per_step=round(pick_ms / pick_n, 3),
                       cross_ms_per_step=round(cross_ms / cross_n, 3))
        if prof["k_sites_own"][1]:
            out.update(own_sort_ms=round(prof["k_sites_own_sort"][0], 3), own_join_ms=round(prof["k_sites_own"][0], 3))
        return out
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--targets", type=int, default=65536)
    ap.add_argument("--pairs", type=int, default=2048)
    args = ap.parse_args()
    import torch
    from multiprime_b200 import _lib, synth
    from multiprime_b200 import primer_coverage as pc
    torch.cuda.set_device(0)
    ctx = _lib.Context.shared(0)
    tmp = tempfile.mkdtemp(prefix="mpb_select_specific_")
    try:
        fa, bgfa = os.path.join(tmp, "targets.fa"), os.path.join(tmp, "background.fa")
        synth.write_pcr_targets(fa, args.targets)
        n_bg = synth.write_pcr_background(bgfa)
        pairs = synth.pcr_candidate_pool(args.pairs)
        sampler = ClockSampler(0)
        sampler.start()
        build = run_build(ctx, pc.read_targets(fa), pairs, args.steps, args.warmup)
        tools = [run_tool(ctx, fa, bgfa, pairs, args.steps, args.warmup, f)
                 for f in ({}, {"cross": True}, {"background": True}, {"cross": True, "background": True})]
        sampler.stop_flag.set()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps({"metric": "select_specific_e2e_s", "value": tools[3]["e2e_s_median"], "unit": "s", "n_gpus": 1,
                      "steps": args.steps, "warmup": args.warmup, "higher_is_better": False, "data": "synthetic",
                      "v": V, "size": list(SIZE), "background_records": n_bg, "build": build, "tool": tools,
                      "device": torch.cuda.get_device_name(0), "clocks": sampler.summary()}))
