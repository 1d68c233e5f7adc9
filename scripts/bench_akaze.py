"""Fast-AKAZE detection throughput on one GPU (r3d_akaze_detect) with parity against the CPU restatement.

    python scripts/bench_akaze.py [--images 32] [--width 4000] [--height 3000] [--reps 3] [--parity 2]

Seeded procedural images (tests/akaze_scenes.py).  Prints one JSON line: images/s and keypoints/s of the whole call
(host clock around calls that end in a device synchronise, after a warm-up call on the same shapes), the per-stage
device times of the last call (CUDA events), the bytes the scale space moves per image from the level shapes and the
FED step counts against the card's HBM bandwidth, and parity with the oracle on the first --parity images.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from akaze_scenes import scene  # noqa: E402
from regard3d_b200 import capi  # noqa: E402


def scale_space_bytes(w, h):
    """DRAM bytes the scale-space kernels read and write for one image, counting every plane pass once per read and
    once per write (float32): blur / Scharr / Hessian passes are 2 plane reads + 2 writes each (row pass into the
    scratch plane, column pass out), FED sweeps 2 reads + 1 write (step) and 2 reads + 1 write (update)."""
    lv = capi.akaze_levels(w, h)
    total = 0
    for i, l in enumerate(lv):
        px = int(l["width"]) * int(l["height"]) * 4
        sep_passes = 1 + 5 + (3 if i else 0) + (3 if i == 0 and len(lv) > 1 else 0)  # blur, Hessian, (blur + Scharr)
        total += sep_passes * 4 * px + 3 * px  # + Ldet: 3 reads, 1 write (approx.)
        if i:
            total += 2 * px + 3 * px  # Lt copy / halving, conductivity
            total += int(l["n_tau"]) * 6 * px
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--width", type=int, default=4000)
    ap.add_argument("--height", type=int, default=3000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--parity", type=int, default=2)
    ap.add_argument("--threshold", type=float, default=1e-3)
    a = ap.parse_args()
    imgs = [scene(a.width, a.height, seed=100 + i) for i in range(a.images)]
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    ctx = capi.Context((0,))
    ctx.akaze_detect(imgs[:2], threshold=a.threshold)  # warm-up: module load, pool blocks
    times = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        got = ctx.akaze_detect(imgs, threshold=a.threshold)
        times.append(time.perf_counter() - t0)
    st = ctx.akaze_timing()
    n_kp = sum(len(k) for k in got)
    best = min(times)
    parity = True
    cpu_s = 0.0
    if a.parity:
        from oracle import pyoracle_akaze as pa
        for i in range(a.parity):
            t0 = time.perf_counter()
            exp = pa.detect(imgs[i], a.threshold)
            cpu_s += time.perf_counter() - t0
            parity &= exp.tobytes() == got[i].tobytes()
    bpi = scale_space_bytes(a.width, a.height)
    ss_s = st["scale_space_ms"] / 1e3
    out = {
        "workload": "akaze_detect", "gpu": gpu[0] if gpu else "unknown", "images": a.images,
        "shape": [a.width, a.height], "threshold": a.threshold, "reps": a.reps,
        "call_s": [round(t, 4) for t in times], "images_per_s": a.images / best, "keypoints": n_kp,
        "keypoints_per_s": n_kp / best, "stage_ms": {k: round(st[k], 3) for k in (
            "scale_space_ms", "candidates_ms", "same_level_ms", "cross_level_ms", "refine_orient_ms")},
        "batches": st["batches"], "kernel_launches": st["kernel_launches"],
        "scale_space_bytes_per_image": bpi, "scale_space_GBps": bpi * a.images / ss_s / 1e9 if ss_s else None,
        "scale_space_share_of_3350GBps": bpi * a.images / ss_s / 3.35e12 if ss_s else None,
        "cpu_restatement_s_per_image": cpu_s / a.parity if a.parity else None, "parity": bool(parity),
    }
    ctx.close()
    print(json.dumps(out))
    return 0 if parity else 1


if __name__ == "__main__":
    sys.exit(main())
