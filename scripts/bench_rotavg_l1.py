"""Global rotations by the L1 method (r3d_rotation_averaging_l1) on one GPU, against the CPU restatement.

    python scripts/bench_rotavg_l1.py [--views 300] [--steps 5] [--warmup 1] [--noise 0.5] [--outliers 0.1]

Input: the problem of bench_rotavg.py (a complete graph over N views, uniform ground-truth rotations, 0.5 degree noise
per edge, 10 % of the edges replaced by random rotations), built directly as r3d_relative_pose records.  GPU arm: the
whole call (median of --steps after --warmup), the stage times and iteration counts of its summary.  CPU arm:
tests/rotavg_l1_ref.py on the same problem (numpy / LAPACK with all usable CPUs); parity compares the two (identical
support / kept sets, iteration counts and termination, rotations within 1e-8).  Also the largest angle of either
result from the truth.  Prints one JSON line.  Writes nothing.
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
    import rotavg_l1_ref as ref
    from bench_relpose import gpu_info
    from regard3d_b200 import build, capi
    from rotavg_scenes import complete_edges, gauge_error_fro, make_problem
    build.build()
    rel, Rs, _ = make_problem(a.views, complete_edges(a.views), noise_deg=a.noise, outlier_frac=a.outliers, seed=a.seed,
                              outlier_min_deg=0.0)
    ctx = capi.Context((0,))
    for _ in range(a.warmup):
        ctx.rotation_averaging_l1(rel, a.views)
    times = []
    for _ in range(a.steps):
        t0 = time.perf_counter()
        got = ctx.rotation_averaging_l1(rel, a.views)
        times.append(time.perf_counter() - t0)
    S = got[4]
    n_thr = len(os.sched_getaffinity(0))
    t0 = time.perf_counter()
    exp = ref.rotation_averaging_l1(rel, a.views)
    cpu_s = time.perf_counter() - t0
    E = exp[4]
    iters = ("l1_iterations", "pd_iterations", "pd_backtracks", "irls_iterations", "termination")
    parity = bool(S["success"] == E["success"] and np.array_equal(got[1], exp[1]) and np.array_equal(got[2], exp[2])
                  and np.array_equal(got[3], exp[3]) and S["n_valid_triplets"] == E["n_valid_triplets"]
                  and all(S[k] == E[k] for k in iters) and np.abs(got[0] - exp[0]).max() <= 1e-8)
    deg = lambda r, k: float(np.degrees(gauge_error_fro(r, Rs, k) / np.sqrt(2)))
    med = float(np.median(times))
    res = {"metric": "rotavg_l1_s", "views": a.views, "edges": len(rel), "triplets": int(S["n_triplets"]),
           "valid_triplets": int(S["n_valid_triplets"]), "kept_edges": int(S["n_kept_edges"]),
           "gpu_s_median": med, "gpu_s_all": times,
           "stages_ms": {k: S[k] for k in ("ms_triplets", "ms_init", "ms_l1", "ms_irls", "ms_device_total", "ms_host")},
           **{k: S[k] for k in iters}, "max_rotation_diff": float(np.abs(got[0] - exp[0]).max()),
           "gpu_err_deg": deg(got[0], got[1]), "cpu_err_deg": deg(exp[0], exp[1]),
           "cpu_s": cpu_s, "cpu_threads": n_thr, "cpu_over_gpu": cpu_s / med, "parity": parity}
    res.update(gpu_info())
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
