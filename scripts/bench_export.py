"""What follows the SfM engine on one GPU: the undistortion of every view (r3d_undistort_images) and the colour plan
(r3d_sfm_colorize_plan), each against the CPU restatement (oracle/oracle_export.cpp).

    python scripts/bench_export.py [--views 32] [--width 4000] [--height 3000] [--steps 3] [--warmup 1] [--cpu-images 2]

Undistortion, for radial K3 and for the fisheye: --views random RGB images of width x height, one call per step (median
of --steps after --warmup).  Reported: the kernels' device time and their effective bandwidth (each image read once and
written once), the upload / download / staging times, images per second end to end (pageable numpy arrays in and out, as
a caller holds them), and the single-threaded CPU restatement's time per image on the first --cpu-images of the same
images, whose outputs must equal the GPU's byte for byte.  Colour plan: the scene of bench.py's bundle-adjustment leg
(synth.make_ba_problem(200, 200000, 5), about 10^6 observations) as an SfmData; the device call's time (median) against
the oracle's, and parity of the three outputs.  Prints one JSON line.  Writes nothing.
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

MODELS = {"radial3": (3, (-0.12, 0.05, -0.01)), "fisheye": (5, (0.03, -0.01, 0.004, -0.001))}


def undistort_leg(ctx, a, pe):
    rng = np.random.default_rng(3)
    imgs = [rng.integers(0, 256, size=(a.height, a.width, 3), dtype=np.uint8) for _ in range(a.views)]
    out = {}
    for name, (model, disto) in MODELS.items():
        f = 1.1 * max(a.width, a.height)
        intr = [dict(model=model, focal=f, ppx=a.width / 2.0, ppy=a.height / 2.0, disto=disto)] * a.views
        for _ in range(a.warmup):
            ctx.undistort_images(intr, imgs)
        walls, timings = [], []
        for _ in range(a.steps):
            t0 = time.perf_counter()
            got = ctx.undistort_images(intr, imgs)
            walls.append(time.perf_counter() - t0)
            timings.append(ctx.last_undistort_timing)
        k = int(np.argsort(walls)[len(walls) // 2])
        t = timings[k]
        img_bytes = a.width * a.height * 3
        t_cpu, parity = [], True
        for i in range(min(a.cpu_images, a.views)):
            t0 = time.perf_counter()
            ref = pe.undistort_image(model, f, a.width / 2.0, a.height / 2.0, disto, imgs[i])
            t_cpu.append(time.perf_counter() - t0)
            parity &= bool(np.array_equal(ref, got[i]))
        black = float((got[0].reshape(-1, 3) == 0).all(-1).mean())
        out[name] = {"wall_s_median": walls[k], "wall_s_all": walls, "images_per_s": a.views / walls[k],
                     "kernel_ms": t["kernel_ms"], "kernel_ms_per_image": t["kernel_ms"] / a.views,
                     "kernel_effective_GBps": 2.0 * img_bytes * a.views / (t["kernel_ms"] * 1e-3) / 1e9,
                     "upload_ms": t["upload_ms"], "download_ms": t["download_ms"], "stage_ms": t["stage_ms"],
                     "pcie_GBps_up": img_bytes * a.views / (t["upload_ms"] * 1e-3) / 1e9,
                     "pcie_GBps_down": img_bytes * a.views / (t["download_ms"] * 1e-3) / 1e9,
                     "cpu_s_per_image": float(np.median(t_cpu)) if t_cpu else None, "cpu_images": len(t_cpu),
                     "cpu_over_gpu_per_image": float(np.median(t_cpu)) / (walls[k] / a.views) if t_cpu else None,
                     "black_fraction": black, "parity": parity}
    return out


def plan_leg(ctx, a, capi, pe):
    from export_scenes import to_sfm
    from regard3d_b200 import synth
    w, h = 1920, 1080
    p = synth.make_ba_problem(n_cams=200, n_pts=200000, obs_per_pt=5, seed=20260924 + 5, w=w, h=h)
    n_lm = len(p["points"])
    xy = p["obs_xy"].reshape(n_lm, 5, 2)
    xy[..., 0] = np.clip(xy[..., 0], 0.0, w - 1.0)
    xy[..., 1] = np.clip(xy[..., 1], 0.0, h - 1.0)
    cam = p["obs_cam"].reshape(n_lm, 5)
    views = [dict(id_view=v, width=w, height=h, has_pose=True) for v in range(200)]
    landmarks = [dict(id=l, X=p["points"][l].tolist(),
                      obs=sorted((int(c), k, float(xy[l, k, 0]), float(xy[l, k, 1])) for k, c in enumerate(cam[l].tolist())))
                 for l in range(n_lm)]
    sd = to_sfm(capi, views, landmarks)
    for _ in range(a.warmup):
        ctx.colorize_plan(sd)
    times = []
    for _ in range(a.steps):
        t0 = time.perf_counter()
        got = ctx.colorize_plan(sd)
        times.append(time.perf_counter() - t0)
    flat = pe.flatten(views, landmarks)
    t0 = time.perf_counter()
    exp = pe.colorize_plan(*flat)
    cpu_s = time.perf_counter() - t0
    med = float(np.median(times))
    return {"landmarks": n_lm, "observations": int(5 * n_lm), "views": 200, "rounds": int(len(got[0])),
            "gpu_s_median": med, "gpu_s_all": times, "cpu_s": cpu_s, "cpu_over_gpu": cpu_s / med,
            "parity": bool(all(np.array_equal(g, e) for g, e in zip(got, exp)))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=32)
    ap.add_argument("--width", type=int, default=4000)
    ap.add_argument("--height", type=int, default=3000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--cpu-images", type=int, default=2)
    a = ap.parse_args()
    from bench_relpose import gpu_info
    from oracle import pyoracle_export as pe
    from regard3d_b200 import build, capi
    build.build()
    pe.build()
    ctx = capi.Context((0,))
    res = {"metric": "export", "views": a.views, "width": a.width, "height": a.height,
           "host_threads": len(os.sched_getaffinity(0)), "undistort": undistort_leg(ctx, a, pe),
           "colorize_plan": plan_leg(ctx, a, capi, pe)}
    res.update(gpu_info())
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
