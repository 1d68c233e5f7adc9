"""Global translations by the L-infinity translation LP (r3d_translation_averaging_l1, Regard3D's default L1 method) on
one GPU, against the CPU restatement and HiGHS.

    python scripts/bench_transavg_l1.py [--views 300] [--steps 5] [--warmup 1] [--noise 0.5] [--no-highs]

Input: bench_transavg.py's problem, a complete graph over N views (N = 300: 44 850 edges; an LP of 313 950 rows and
45 748 variables, a reduced system of 898) with the true rotations as the global ones and 0.5 degree direction noise.
GPU arm: the whole call (median of --steps after --warmup), the stage times of its summary, the iterations and gamma.
CPU arm: tests/transavg_l1_ref.py (numpy / scipy, the same method) with all usable CPUs.  HiGHS arm:
scipy.optimize.linprog(method="highs-ipm") on the same LP (HiGHS' interior point with crossover to a vertex; its
default choice takes far longer here), as a stand-in for the CLP solver upstream calls (not CLP).
Parity: identical kept sets, both converged, gamma within 2e-9 (1 + gamma) of the restatement's and 1e-9 of HiGHS'.
Prints one JSON line.  Writes nothing.
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
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--no-highs", action="store_true")
    a = ap.parse_args()
    from bench_relpose import gpu_info
    from regard3d_b200 import build, capi
    from scipy.optimize import linprog
    import transavg_l1_ref as ref
    from transavg_scenes import complete_edges, make_problem
    build.build()
    rel, Rs, _, _ = make_problem(a.views, complete_edges(a.views), noise_deg=a.noise, seed=a.seed)
    rk = np.ones(a.views, bool)
    ctx = capi.Context((0,))
    res = {"metric": "transavg_l1_s", "views": a.views, "edges": len(rel), "cpu_threads": len(os.sched_getaffinity(0))}
    for _ in range(a.warmup):
        ctx.translation_averaging_l1(rel, Rs, rk, a.views)
    times = []
    for _ in range(a.steps):
        t0 = time.perf_counter()
        got = ctx.translation_averaging_l1(rel, Rs, rk, a.views)
        times.append(time.perf_counter() - t0)
    S = got[5]
    med = float(np.median(times))
    res["gpu_arm"] = {"s_median": med, "s_all": times, "stages_ms": {k: S[k] for k in ("ms_solve", "ms_device_total", "ms_host")},
                  "iterations": S["iterations"], "regularized_factorizations": S["regularized_factorizations"],
                  "termination": S["termination"], "gamma": S["gamma"], "kept_edges": int(S["n_kept_edges"])}
    t0 = time.perf_counter()
    exp = ref.translation_averaging_l1(rel, Rs, rk, a.views)
    cpu_s = time.perf_counter() - t0
    E = exp[5]
    res["cpu_restatement"] = {"s": cpu_s, "iterations": E["iterations"], "termination": E["termination"], "gamma": E["gamma"],
                              "over_gpu": cpu_s / med}
    parity = bool(S["success"] == E["success"] and np.array_equal(got[2], exp[2]) and np.array_equal(got[3], exp[3])
                  and S["termination"] == 0 and E["termination"] == 0
                  and abs(S["gamma"] - E["gamma"]) <= 2e-9 * (1.0 + E["gamma"]))
    if not a.no_highs:
        G, h, c, _, _ = ref.build_lp(rel, Rs, got[2], got[3])
        t0 = time.perf_counter()
        r = linprog(c, A_ub=G, b_ub=h, bounds=[(None, None)] * G.shape[1], method="highs-ipm")
        hs = time.perf_counter() - t0
        res["highs_stand_in_for_clp"] = {"s": hs, "status": int(r.status), "gamma": float(r.fun), "over_gpu": hs / med}
        parity = parity and r.status == 0 and abs(S["gamma"] - r.fun) <= 1e-9 * max(1.0, r.fun)
    res["parity"] = parity
    res.update(gpu_info())
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
