#!/usr/bin/env python
"""Pool-assignment benchmark (primer_pools.py; DESIGN.md §4, profiles/h100_bench_pools.json); prints one JSON line.

    python tools/bench_pools.py --steps 3 --warmup 1 [--targets 65536]

search  mpb_pool_search alone on planted instances of 512 pairs (conflicts only across a hidden balanced partition,
        5 % of the other pairs, weights 1..12) in P = 2, 8, 32 pools, with the tool's default restarts and iterations:
        kernel ms per call from CUDA events; steps run (a restart that reaches cost 0 stops there); steps/s and candidate
        evaluations/s (the evaluations per step taken from the CPU double's run of restart 0); the best cost and the
        step that reached it; the CPU double's seconds for restart 0 on one core, for contrast.
tool    the panel and targets of tools/bench_specificity.py (48 tiled pairs, v = 3, -s 50,2000, 65 536 synthetic
        targets) split into P = 2, 4, 8 pools: the cost, the time of the specificity call, the dimer grid and the
        search, and the end-to-end time from the FASTA file.
The card's name, SM clock and enforced power limit are recorded the way bench.py records them."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler  # noqa: E402


def planted(n, P, seed, density=0.05):
    import numpy as np
    rng = np.random.default_rng(seed)
    hidden = rng.permutation(np.arange(n) % P)
    w = np.triu(rng.integers(1, 13, (n, n)) * (rng.random((n, n)) < density), 1)
    w = w + w.T
    w[hidden[:, None] == hidden[None, :]] = 0
    return w.astype(np.uint8)


def double_restart0(w, P, seed, iterations):
    """(seconds, steps, candidate evaluations) of restart 0 on the CPU double"""
    import numpy as np
    from tests import fake_pool_search as fps
    n = len(w)
    W = w.astype(np.int64)
    evals = [0]

    def trace(t, pool, cost):
        same = pool[:, None] == pool[None, :]
        K = int(((W * same).sum(axis=1) > 0).sum())
        if cost > 0:
            evals[0] += K * n + (K * P if n % P else 0)
    t0 = time.perf_counter()
    fps.restart_search(w, P, seed, 0, iterations)
    sec = time.perf_counter() - t0
    steps = [0]

    def count(t, pool, cost):
        steps[0] = t
        trace(t, pool, cost)
    fps.restart_search(w, P, seed, 0, iterations, count)
    return sec, steps[0], evals[0]


def run_search(args, ctx):
    from multiprime_b200 import primer_pools as pp
    out = {}
    for P in (2, 8, 32):
        w = planted(512, P, 2024 + P)
        for _ in range(args.warmup):
            res = ctx.pool_search(w, P, pp.SEED, 0, pp.RESTARTS, pp.ITERATIONS)
        ctx.profile_read(None)
        ctx.profile(True)
        for _ in range(args.steps):
            res = ctx.pool_search(w, P, pp.SEED, 0, pp.RESTARTS, pp.ITERATIONS)
        ms, launches, _ = ctx.profile_read("k_pool_search")
        ctx.profile(False)
        ms /= max(1, launches)
        solved = res["cost"] == 0
        steps = int(res["step"][solved].sum()) + pp.ITERATIONS * int((~solved).sum())
        sec0, steps0, evals0 = double_restart0(w, P, pp.SEED, pp.ITERATIONS)
        k = int(res["cost"].argmin())
        out["P%d" % P] = {"kernel_ms": round(ms, 3), "restarts": pp.RESTARTS, "iterations": pp.ITERATIONS,
                          "restarts_at_cost_0": int(solved.sum()), "steps": steps,
                          "steps_per_s": round(steps / (ms / 1000)), "evals_per_step_restart0": round(evals0 / max(1, steps0)),
                          "cand_evals_per_s": round(steps / (ms / 1000) * evals0 / max(1, steps0)),
                          "best_cost": int(res["cost"][k]), "best_step": int(res["step"][k]),
                          "median_best_step": float(statistics.median(res["step"].tolist())),
                          "double_s_restart0_one_core": round(sec0, 3)}
    return out


def run_tool(args):
    import shutil
    import tempfile
    from multiprime_b200 import primer_pools as pp
    from multiprime_b200 import synth
    tmp = tempfile.mkdtemp(prefix="mpb_pools_")
    try:
        fa = os.path.join(tmp, "targets.fa")
        pairs = synth.write_pcr_targets(fa, args.targets)
        out = {}
        pp.run(fa, pairs, os.path.join(tmp, "warm"), 3, "1,2,-1", (50, 2000), 2)
        for P in (2, 4, 8):
            times = {}
            t0 = time.perf_counter()
            res = pp.run(fa, pairs, os.path.join(tmp, "out%d" % P), 3, "1,2,-1", (50, 2000), P, _times=times)
            e2e = time.perf_counter() - t0
            w = res["w"]
            out["P%d" % P] = {"cost": res["cost"], "cost_one_pool": int(w.astype(int).sum()) // 2,
                              "specificity_s": round(times["specificity"], 3), "dimer_s": round(times["dimer"], 3),
                              "search_s": round(times["search"], 3), "e2e_s_from_fasta": round(e2e, 3)}
        return {"pairs": len(pairs), "targets": args.targets, "P": out}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--targets", type=int, default=65536, help="synthetic targets of the whole-tool part")
    args = ap.parse_args()
    import torch
    from multiprime_b200 import _lib
    torch.cuda.set_device(0)
    ctx = _lib.Context.shared(0)
    sampler = ClockSampler(0)
    sampler.start()
    search = run_search(args, ctx)
    tool = run_tool(args)
    sampler.stop_flag.set()
    p8 = search["P8"]
    print(json.dumps({"metric": "pool_search_steps_per_sec", "value": p8["steps_per_s"], "unit": "steps/s",
                      "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "higher_is_better": True,
                      "data": "synthetic", "search_512_pairs": search, "tool": tool,
                      "device": torch.cuda.get_device_name(0), "clocks": sampler.summary()}))
