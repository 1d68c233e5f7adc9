"""Global rotations from relative motions (r3d_rotation_averaging) on one GPU, against the CPU restatement.

    python scripts/bench_rotavg.py [--views 300] [--steps 5] [--warmup 1] [--noise 0.5] [--outliers 0.1]

Input: synthetic relative poses, built directly as r3d_relative_pose records (no matching): a complete graph over N
views with uniform (non-commuting) ground-truth rotations, 0.5 degree rotation noise per edge and 10 % of the edges
replaced by random rotations.  GPU arm: the whole call (median of --steps after --warmup), the stage times of its
summary and the triplet count.  CPU arm: orc_rotation_averaging on the same problem with all usable CPUs; parity
compares the two (identical support / kept sets and LM iteration count, rotations within 1e-8).  Prints one JSON line.
Writes nothing.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=300)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--noise", type=float, default=0.5)
    ap.add_argument("--outliers", type=float, default=0.1)
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    from bench_relpose import gpu_info
    from oracle import pyoracle_rotavg as por
    from regard3d_b200 import build, capi
    from rotavg_scenes import complete_edges, make_problem
    build.build()
    rel, _, _ = make_problem(a.views, complete_edges(a.views), noise_deg=a.noise, outlier_frac=a.outliers, seed=a.seed,
                             outlier_min_deg=0.0)
    ctx = capi.Context((0,))
    for _ in range(a.warmup):
        ctx.rotation_averaging(rel, a.views)
    times = []
    for _ in range(a.steps):
        t0 = time.perf_counter()
        got = ctx.rotation_averaging(rel, a.views)
        times.append(time.perf_counter() - t0)
    S = got[4]
    n_thr = len(os.sched_getaffinity(0))
    t0 = time.perf_counter()
    exp = por.rotation_averaging(rel, a.views, n_threads=n_thr)
    cpu_s = time.perf_counter() - t0
    E = exp[4]
    parity = bool(S["success"] == E["success"] and np.array_equal(got[1], exp[1]) and np.array_equal(got[2], exp[2])
                  and np.array_equal(got[3], exp[3]) and S["n_triplets"] == E["n_triplets"]
                  and S["n_valid_triplets"] == E["n_valid_triplets"] and S["lm_iterations"] == E["lm_iterations"]
                  and S["lm_termination"] == E["lm_termination"] and np.abs(got[0] - exp[0]).max() <= 1e-8)
    med = float(np.median(times))
    res = {"metric": "rotavg_s", "views": a.views, "edges": len(rel), "triplets": int(S["n_triplets"]),
           "valid_triplets": int(S["n_valid_triplets"]), "kept_edges": int(S["n_kept_edges"]),
           "gpu_s_median": med, "gpu_s_all": times,
           "stages_ms": {k: S[k] for k in ("ms_triplets", "ms_init", "ms_refine", "ms_device_total", "ms_host")},
           "init_iterations": S["init_iterations"], "lm_iterations": S["lm_iterations"],
           "cpu_s": cpu_s, "cpu_threads": n_thr, "cpu_over_gpu": cpu_s / med, "parity": parity}
    res.update(gpu_info())
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
