"""Keypoint detection throughput on one GPU (r3d_detect_keypoints) with parity against the CPU restatement.

    python scripts/bench_akaze.py [--detector fast-akaze|akaze] [--images 32] [--width 4000] [--height 3000]
                                  [--reps 3] [--parity 2]

Seeded procedural images (tests/akaze_scenes.py).  Prints one JSON line: images/s and keypoints/s of the whole call
(host clock around calls that end in a device synchronise, after a warm-up call on the same shapes), the per-stage
device times of the last call (CUDA events), the bytes the scale space moves per image from the level shapes and the
FED step counts against the card's HBM bandwidth, and parity with the restatement on the first --parity images
(oracle/oracle_akaze.cpp for Fast-AKAZE, tests/akaze_cv_ref.py for AKAZE).  With --detector akaze and cv2 importable,
cv2.AKAZE_create(...).detect -- the reference's own detector -- is also timed on the same parity images, with
cv2.getNumThreads() recorded.
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
    ap.add_argument("--detector", choices=("fast-akaze", "akaze"), default="fast-akaze")
    a = ap.parse_args()
    det = capi.DETECTOR_AKAZE if a.detector == "akaze" else capi.DETECTOR_FAST_AKAZE
    imgs = [scene(a.width, a.height, seed=100 + i) for i in range(a.images)]
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    ctx = capi.Context((0,))
    ctx.akaze_detect(imgs[:2], detector=det, threshold=a.threshold)  # warm-up: module load, pool blocks
    times = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        got = ctx.akaze_detect(imgs, detector=det, threshold=a.threshold)
        times.append(time.perf_counter() - t0)
    st = ctx.akaze_timing()
    n_kp = sum(len(k) for k in got)
    best = min(times)
    parity = True
    cpu_s = 0.0
    cv2_s, cv2_kp, cv2_threads = None, None, None
    if a.parity:
        if det == capi.DETECTOR_AKAZE:
            import akaze_cv_ref
            restated = akaze_cv_ref.detect
        else:
            from oracle import pyoracle_akaze as pa
            restated = pa.detect
        for i in range(a.parity):
            t0 = time.perf_counter()
            exp = restated(imgs[i], a.threshold)
            cpu_s += time.perf_counter() - t0
            parity &= exp.tobytes() == got[i].tobytes()
        try:
            import cv2
        except ImportError:
            cv2 = None
        if cv2 is not None and det == capi.DETECTOR_AKAZE:
            d = cv2.AKAZE_create(cv2.AKAZE_DESCRIPTOR_MLDB, 0, 3, a.threshold, 4, 4, cv2.KAZE_DIFF_PM_G2)
            d.detect(imgs[0][:480, :640], None)
            t0 = time.perf_counter()
            cv2_kp = sum(len(d.detect(imgs[i], None)) for i in range(a.parity))
            cv2_s = (time.perf_counter() - t0) / a.parity
            cv2_threads = cv2.getNumThreads()
    bpi = scale_space_bytes(a.width, a.height)
    ss_s = st["scale_space_ms"] / 1e3
    out = {
        "workload": "akaze_detect", "detector": a.detector, "gpu": gpu[0] if gpu else "unknown", "images": a.images,
        "shape": [a.width, a.height], "threshold": a.threshold, "reps": a.reps,
        "call_s": [round(t, 4) for t in times], "images_per_s": a.images / best, "keypoints": n_kp,
        "keypoints_per_s": n_kp / best, "stage_ms": {k: round(st[k], 3) for k in (
            "scale_space_ms", "candidates_ms", "same_level_ms", "cross_level_ms", "refine_orient_ms")},
        "batches": st["batches"], "kernel_launches": st["kernel_launches"],
        "scale_space_bytes_per_image": bpi, "scale_space_GBps": bpi * a.images / ss_s / 1e9 if ss_s else None,
        "scale_space_share_of_3350GBps": bpi * a.images / ss_s / 3.35e12 if ss_s else None,
        "cpu_restatement_s_per_image": cpu_s / a.parity if a.parity else None, "parity": bool(parity),
        "cv2_detect_s_per_image": cv2_s, "cv2_keypoints": cv2_kp, "cv2_threads": cv2_threads,
    }
    ctx.close()
    print(json.dumps(out))
    return 0 if parity else 1


if __name__ == "__main__":
    sys.exit(main())
