"""Global translations from relative motions and global rotations (r3d_translation_averaging) on one GPU, against the CPU
restatement, for both methods (L2 chordal and soft-L1).

    python scripts/bench_transavg.py [--views 300] [--steps 5] [--warmup 1] [--noise 0.5]

Input: synthetic relative poses, built directly as r3d_relative_pose records (no matching): a complete graph over N
views (N = 300: 44 850 edges) with uniform ground-truth centres and rotations, the true rotations as the global ones,
and relative translation directions turned by 0.5 degree noise.  GPU arm: the whole call (median of --steps after
--warmup) and the stage times of its summary.  CPU arm: orc_translation_averaging on the same problem with all usable
CPUs.  Parity: identical kept sets, LM iterations and termination, centres and translations within 1e-8 of the scene
scale.  Prints one JSON line.  Writes nothing.
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
    a = ap.parse_args()
    from bench_relpose import gpu_info
    from oracle import pyoracle_transavg as pto
    from regard3d_b200 import build, capi
    from transavg_scenes import complete_edges, make_problem
    build.build()
    rel, Rs, _, _ = make_problem(a.views, complete_edges(a.views), noise_deg=a.noise, seed=a.seed)
    rk = np.ones(a.views, bool)
    ctx = capi.Context((0,))
    n_thr = len(os.sched_getaffinity(0))
    res = {"metric": "transavg_s", "views": a.views, "edges": len(rel), "cpu_threads": n_thr}
    parity_all = True
    for name, method in (("chordal", capi.TRANSAVG_L2_CHORDAL), ("softl1", capi.TRANSAVG_SOFTL1)):
        for _ in range(a.warmup):
            ctx.translation_averaging(rel, Rs, rk, a.views, method=method)
        times = []
        for _ in range(a.steps):
            t0 = time.perf_counter()
            got = ctx.translation_averaging(rel, Rs, rk, a.views, method=method)
            times.append(time.perf_counter() - t0)
        S = got[4]
        t0 = time.perf_counter()
        exp = pto.translation_averaging(rel, Rs, rk, a.views, method=method, n_threads=n_thr)
        cpu_s = time.perf_counter() - t0
        E = exp[4]
        scale = max(np.abs(exp[0]).max(), np.abs(exp[1]).max(), 1e-300)
        parity = bool(S["success"] == E["success"] and np.array_equal(got[2], exp[2]) and np.array_equal(got[3], exp[3])
                      and S["lm_iterations"] == E["lm_iterations"] and S["lm_termination"] == E["lm_termination"]
                      and np.abs(got[0] - exp[0]).max() <= 1e-8 * scale and np.abs(got[1] - exp[1]).max() <= 1e-8 * scale)
        parity_all = parity_all and parity
        med = float(np.median(times))
        res[name] = {"gpu_s_median": med, "gpu_s_all": times,
                     "stages_ms": {k: S[k] for k in ("ms_solve", "ms_device_total", "ms_host")},
                     "lm_iterations": S["lm_iterations"], "lm_termination": S["lm_termination"],
                     "kept_edges": int(S["n_kept_edges"]), "cpu_s": cpu_s, "cpu_over_gpu": cpu_s / med, "parity": parity}
    res["parity"] = parity_all
    res.update(gpu_info())
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
