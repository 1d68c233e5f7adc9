"""Resection of a batch of views (r3d_resect_views) on one GPU, against the CPU restatement.

    python scripts/bench_resection.py [--views 200] [--corr 5000] [--outliers 0.3] [--steps 3] [--warmup 1] [--sample 16]

Scene: what one round of the incremental engine that resects every remaining view hands over: seeded views
(tests/resection_scenes.py) of --corr 2D-3D correspondences each, radial-K3 intrinsics with distortion, 0.3 px noise, a
fraction of outliers; default options (4096 iterations, a-contrario precision, pose refinement on).  The timed region is
the whole call, host clock around it (it ends in a device synchronise and returns host results); the AC-RANSAC /
refinement split comes from CUDA events around the kernels.  The CPU arm is orc_resect_views (OpenMP over views, all
usable CPUs) on a seeded sample of the views; "parity" compares the two on that sample.  Prints one JSON line.  Writes
nothing.  Needs a GPU: creating the context fails without one.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    """Card name and power limit, read-only query."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clk = [s.strip() for s in out[0].split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:  # noqa: BLE001
        return {"gpu": "unknown (%s)" % e}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=200)
    ap.add_argument("--corr", type=int, default=5000)
    ap.add_argument("--outliers", type=float, default=0.3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=16)
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    from regard3d_b200 import capi
    from oracle import pyoracle_resection as pro
    from resection_scenes import make_batch
    ctx = capi.Context((0,))
    views = make_batch(a.seed, a.views, a.corr, models=(3,), outliers=a.outliers)
    counts = [a.corr] * a.views
    X = np.concatenate([v["X"] for v in views])
    x = np.concatenate([v["x"] for v in views])
    cols = {k: [v[k] for v in views] for k in ("width", "height", "model", "focal", "ppx", "ppy", "disto")}
    rv = capi.resection_views(counts, cols["width"], cols["height"], cols["model"], cols["focal"], cols["ppx"], cols["ppy"],
                              cols["disto"])
    for _ in range(a.warmup):
        ctx.resect_views(rv, X, x)
    times = []
    for _ in range(a.steps):
        t0 = time.perf_counter()
        got, gofs, ginl = ctx.resect_views(rv, X, x)
        times.append(time.perf_counter() - t0)
    timing = ctx.resection_timing()
    rng = np.random.default_rng(a.seed)
    sel = np.sort(rng.choice(a.views, min(a.sample, a.views), replace=False))
    n_thr = len(os.sched_getaffinity(0))
    intrs = np.array([pro.intr8(views[v]["focal"], views[v]["ppx"], views[v]["ppy"], views[v]["disto"]) for v in sel])
    t0 = time.perf_counter()
    exp, eofs, einl = pro.resect_views(sel.astype(np.uint64) * a.corr, [a.corr] * len(sel), [cols["width"][v] for v in sel],
                                       [cols["height"][v] for v in sel], [3] * len(sel), intrs, X, x, n_threads=n_thr)
    cpu_s = time.perf_counter() - t0
    parity = True
    for k, v in enumerate(sel):
        g, e = got[v], exp[k]
        parity &= bool(g["status"] == e["status"] and np.array_equal(g["rotation_ransac"], e["rotation_ransac"])
                       and np.array_equal(g["translation_ransac"], e["translation_ransac"])
                       and np.array_equal(ginl[int(gofs[v]):int(gofs[v + 1])], einl[int(eofs[k]):int(eofs[k + 1])]))
        if e["status"] == pro.RESECT_OK:
            parity &= bool(g["lm_iterations"] == e["lm_iterations"] and g["lm_termination"] == e["lm_termination"]
                           and abs(g["lm_final_cost"] - e["lm_final_cost"]) <= 1e-8 * e["lm_final_cost"])
    med = float(np.median(times))
    res = {"metric": "resection_views_per_s", "views": a.views, "correspondences_per_view": a.corr, "outliers": a.outliers,
           "ok_views": int((got["status"] == 0).sum()), "gpu_views_per_s": a.views / med, "gpu_s_median": med, "gpu_s_all": times,
           "resection_timing": timing, "cpu_views_per_s": len(sel) / cpu_s, "cpu_threads": n_thr,
           "cpu_sample_views": int(len(sel)), "parity": parity, "lm_iterations_mean": float(got["lm_iterations"].mean())}
    res.update(gpu_info())
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
