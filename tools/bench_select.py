#!/usr/bin/env python
"""Greedy set-selection benchmark (primer_select.py; DESIGN.md §4, profiles/h100_bench_select.json); prints one JSON
line.

    python tools/bench_select.py --steps 3 --warmup 1 [--targets 65536] [--pairs 2048]

Workload: the targets of synth.write_pcr_targets (unchanged) and a pool of --pairs candidates from
synth.pcr_candidate_pool; v = 3, -c 1,2,-1, -s 50,2000, the tool's defaults otherwise.
cover    the matrix build (mpb_pattern_cover in blocks of pairs): per call search / filter / sort / join ms from CUDA
         events, the k_pattern_sites launches per build (one per call when the capacity held the sites) and ms per
         launch, sites; the build's wall time.
gains    the greedy's mpb_cover_gains calls in a tool run (ms per step, bytes of the listed rows per step over kernel
         time), and the kernel alone over every row of the pool's matrix and of a 16 384-pair x 65 536-target matrix
         (268 MB, larger than the L2), against the 3.35 TB/s of the H100 SXM data sheet.
tool     steps taken, final coverage, the dimer grid, and the whole tool from the FASTA file to its three output files.
double   the CPU double's matrix build (tests/fake_pattern_cover.py) on a subset, for contrast.
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

HBM_TBS = 3.35
V, SIZE = 3, (50, 2000)


def profiled(ctx, names):
    out = {}
    for n in names:
        ms, launches, units = ctx.profile_read(n)
        out[n] = (ms, launches, units)
    return out


def run_cover(ctx, fa, pairs, steps, warmup):
    """the matrix build alone, profiled: per-call kernel ms and the wall time of the build"""
    import numpy as np
    from multiprime_b200 import _lib
    from multiprime_b200 import primer_coverage as pc
    from multiprime_b200 import primer_select as sel
    targets = pc.read_targets(fa)
    pool = sel.Pool(pairs, {}, "1,2,-1")
    block = sel.block_of(len(targets.names), len(pool.names))
    walls, res = [], None
    for it in range(warmup + steps):
        if it == warmup:
            ctx.profile_read(None)
            ctx.profile(True)
        stats = np.zeros(3, np.int64)
        t0 = time.perf_counter()
        _, mat = sel.build_matrix(targets, pool.panel, V, SIZE[0], SIZE[1], 0, None, _lib, block, stats)
        ctx.sync()
        walls.append(time.perf_counter() - t0)
        if it == warmup + steps - 1:
            amp, perf, _, _ = mat.to_host()
            res = dict(stats=stats, amp_bits=int(np.unpackbits(amp.view(np.uint8)).sum()))
        mat.close()
    prof = profiled(ctx, ["k_pattern_sites", "k_cover_filter", "k_cover_sort", "k_cover_join"])
    ctx.profile(False)
    calls = prof["k_cover_join"][1] or 1
    searches = prof["k_pattern_sites"][1] or 1
    st = res["stats"]
    return {"pairs": len(pairs), "targets": len(targets.names), "block_pairs": block, "calls_per_build": calls // steps,
            "search_launches_per_build": searches // steps,
            "search_ms_per_launch": round(prof["k_pattern_sites"][0] / searches, 2),
            "search_ms_per_call": round(prof["k_pattern_sites"][0] / calls, 2),
            "filter_ms_per_call": round(prof["k_cover_filter"][0] / calls, 2),
            "sort_ms_per_call": round(prof["k_cover_sort"][0] / calls, 2),
            "join_ms_per_call": round(prof["k_cover_join"][0] / calls, 2),
            "search_hits_per_build": int(st[0]), "left_sites": int(st[1]), "right_sites": int(st[2]),
            "amplified_bits": res["amp_bits"], "build_wall_s": [round(w, 3) for w in walls[warmup:]]}, targets


def gains_alone(ctx, n_rows, n_rec, reps):
    """k_cover_gains over every row of an n_rows x n_rec matrix: ms per call and bytes/s"""
    import numpy as np
    from multiprime_b200 import _lib
    mat = _lib.CoverMatrix(ctx, n_rows, n_rec)
    try:
        cand = np.arange(n_rows)
        ctx.cover_gains(mat, cand)
        ctx.profile_read(None)
        ctx.profile(True)
        for _ in range(reps):
            ctx.cover_gains(mat, cand)
        ms, launches, units = ctx.profile_read("k_cover_gains")
        ctx.profile(False)
    finally:
        mat.close()
    ms /= launches
    bps = units / launches / (ms / 1e3)
    return {"rows": n_rows, "targets": n_rec, "bytes_per_call": int(units / launches), "ms_per_call": round(ms, 4),
            "tb_per_s": round(bps / 1e12, 3), "fraction_of_3_35_tb_s": round(bps / 1e12 / HBM_TBS, 3)}


def run_tool(ctx, fa, pairs, steps, warmup):
    from multiprime_b200 import primer_select as sel
    tmp = tempfile.mkdtemp(prefix="mpb_select_out_")
    try:
        e2e, runs = [], []
        for it in range(warmup + steps):
            times = {}
            if it == warmup + steps - 1:             # the last run profiled (end-to-end times from the others)
                ctx.profile_read(None)
                ctx.profile(True)
            t0 = time.perf_counter()
            res = sel.run(fa, pairs, os.path.join(tmp, "o"), V, "1,2,-1", SIZE, _times=times)
            dt = time.perf_counter() - t0
            if it >= warmup:
                e2e.append(dt)
                runs.append(times)
        ms, launches, units = ctx.profile_read("k_cover_gains")
        ctx.profile(False)
        last = runs[-1]
        bps = units / (ms / 1e3) if ms else 0.0
        covered, total = res["covered"], res["total"]
        timed = e2e[:-1] if len(e2e) > 1 else e2e
        return {"steps_taken": last["steps"], "covered": covered, "total": total, "coverage": round(covered / total, 4),
                "gains_calls": launches, "gains_ms_per_call": round(ms / max(1, launches), 4),
                "gains_bytes_per_step": int(units / max(1, launches)), "gains_tb_per_s": round(bps / 1e12, 3),
                "read_s": round(last["read"], 3), "cover_s": round(last["cover"], 3), "dimer_s": round(last["dimer"], 3),
                "greedy_s": round(last["greedy"], 3), "e2e_s_from_fasta": [round(x, 3) for x in timed],
                "e2e_s_median": round(statistics.median(timed), 3)}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def run_double(targets_fa, pairs, n_pairs=4, n_targets=512):
    """the CPU double's matrix build on the first n_targets targets and n_pairs pairs"""
    from multiprime_b200 import primer_coverage as pc
    from multiprime_b200 import primer_select as sel
    from tests import fake_pattern_cover
    tmp = tempfile.mkdtemp(prefix="mpb_select_double_")
    try:
        sub = os.path.join(tmp, "sub.fa")
        with open(targets_fa) as fi, open(sub, "w") as fo:
            for k, line in enumerate(fi):
                if k >= 2 * n_targets:
                    break
                fo.write(line)
        targets = pc.read_targets(sub)
        pool = sel.Pool(dict(list(pairs.items())[:n_pairs]), {}, "1,2,-1")
        t0 = time.perf_counter()
        sel.build_matrix(targets, pool.panel, V, SIZE[0], SIZE[1], 0, None, fake_pattern_cover, n_pairs)
        sec = time.perf_counter() - t0
        return {"pairs": n_pairs, "targets": n_targets, "seconds_one_core": round(sec, 2),
                "pair_targets_per_s": round(n_pairs * n_targets / sec)}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--targets", type=int, default=65536)
    ap.add_argument("--pairs", type=int, default=2048)
    args = ap.parse_args()
    import torch
    from multiprime_b200 import _lib, synth
    torch.cuda.set_device(0)
    ctx = _lib.Context.shared(0)
    tmp = tempfile.mkdtemp(prefix="mpb_select_")
    try:
        fa = os.path.join(tmp, "targets.fa")
        synth.write_pcr_targets(fa, args.targets)
        pairs = synth.pcr_candidate_pool(args.pairs)
        sampler = ClockSampler(0)
        sampler.start()
        cover, targets = run_cover(ctx, fa, pairs, args.steps, args.warmup)
        alone = [gains_alone(ctx, len(pairs), len(targets.names), 50), gains_alone(ctx, 16384, 65536, 20)]
        tool = run_tool(ctx, fa, pairs, max(2, args.steps), args.warmup)
        sampler.stop_flag.set()
        double = run_double(fa, pairs)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps({"metric": "select_e2e_s", "value": tool["e2e_s_median"], "unit": "s", "n_gpus": 1,
                      "steps": args.steps, "warmup": args.warmup, "higher_is_better": False, "data": "synthetic",
                      "v": V, "size": list(SIZE), "cover": cover, "gains_kernel_alone": alone, "tool": tool,
                      "cpu_double": double, "device": torch.cuda.get_device_name(0), "clocks": sampler.summary()}))
