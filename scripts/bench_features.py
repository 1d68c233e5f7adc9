"""Feature extraction throughput on one GPU (r3d_extract_features: Fast-AKAZE + LIOP-144, optionally the .feat / .desc
files) against detection alone and the two-call path, with byte parity of the files against the CPU reference.

    python scripts/bench_features.py [--reps 3] [--parity 2] [--out-dir DIR]

Workloads: the seeded scenes of scripts/bench_akaze.py (tests/akaze_scenes.py), 32 x 4000x3000 and 64 x 640x480.  Per
workload, after a warm-up call on the same shapes, the best of --reps calls of each arm (host clock around calls that
end in a device synchronise):
  detect      ctx.akaze_detect
  two_call    ctx.akaze_detect, then ctx.liop_describe per image (each image uploaded again)
  extract     ctx.extract_features, arrays only
  files       ctx.extract_features writing .feat / .desc into --out-dir (a temporary directory by default, removed after)
The per-stage device times of the last extract call (CUDA events), and how much of the describe time the overlap with
the next batch's scale space hid: describe_ms - (extract - detect - d2h_ms), extract and detect being the library's wall
time of its last call (the Python wall times also include copying every array out of the result), over describe_ms.  CPU arm: the oracle
pipeline (tests/features_ref.py) on the first --parity images, whose files must equal the GPU's byte for byte.
The card's name, power limit and max SM clock are read in the same call.  Prints one JSON line.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from akaze_scenes import scene  # noqa: E402
from regard3d_b200 import capi  # noqa: E402

WORKLOADS = [(32, 4000, 3000), (64, 640, 480)]


def best_of(reps, fn):
    times, out = [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        times.append(time.perf_counter() - t0)
    return min(times), out


def run_workload(ctx, n, w, h, a, out_root):
    imgs = [scene(w, h, seed=100 + i) for i in range(n)]
    names = ["image%06d" % i for i in range(n)]
    out_dir = os.path.join(out_root, "%dx%d" % (w, h))
    os.makedirs(out_dir, exist_ok=True)
    thr = a.threshold
    ctx.akaze_detect(imgs[:2], threshold=thr)  # warm-up: module load, pool blocks
    ctx.extract_features(imgs[:2], threshold=thr)
    t_det, dets = best_of(a.reps, lambda: ctx.akaze_detect(imgs, threshold=thr))
    det_ms = ctx.akaze_timing()["total_ms"]

    def two_call():
        ks = ctx.akaze_detect(imgs, threshold=thr)
        return [ctx.liop_describe(im, np.stack([k["x"], k["y"], k["size"], k["angle"]], 1), 8.0) for im, k in zip(imgs, ks)]

    t_two, _ = best_of(a.reps, two_call)
    t_ext, got = best_of(a.reps, lambda: ctx.extract_features(imgs, threshold=thr))
    st = ctx.extract_timing()
    t_files, _ = best_of(a.reps, lambda: ctx.extract_features(imgs, out_dir=out_dir, basenames=names, threshold=thr))
    st_files = ctx.extract_timing()
    n_kp = sum(len(k) for k, _ in got)
    parity = all(k.tobytes() == d.tobytes() for (k, _), d in zip(got, dets))
    cpu_s = 0.0
    if a.parity:
        import features_ref as fr
        ref_dir = os.path.join(out_root, "ref_%dx%d" % (w, h))
        os.makedirs(ref_dir, exist_ok=True)
        for i in range(min(a.parity, n)):
            t0 = time.perf_counter()
            fr.extract_to(ref_dir, [imgs[i]], [names[i]], thr)
            cpu_s += time.perf_counter() - t0
            for ext in (".feat", ".desc"):
                with open(os.path.join(out_dir, names[i] + ext), "rb") as f1, open(os.path.join(ref_dir, names[i] + ext), "rb") as f2:
                    parity &= f1.read() == f2.read()
    # on the library's own clock (the Python arms also copy every array out of the result); the descriptor download is
    # host time of its own and not part of what the overlap can hide
    hidden = st["describe_ms"] - (st["total_ms"] - det_ms - st["d2h_ms"])
    return {
        "images": n, "shape": [w, h], "threshold": thr, "keypoints": n_kp, "batches": st["batches"],
        "kernel_launches": st["kernel_launches"],
        "call_s": {"detect": round(t_det, 4), "two_call": round(t_two, 4), "extract": round(t_ext, 4),
                   "files": round(t_files, 4)},
        "images_per_s": {"detect": n / t_det, "two_call": n / t_two, "extract": n / t_ext, "files": n / t_files},
        "descriptors_per_s": {"two_call": n_kp / t_two, "extract": n_kp / t_ext, "files": n_kp / t_files},
        "library_ms": {"detect": round(det_ms, 3), "extract": round(st["total_ms"], 3), "files": round(st_files["total_ms"], 3)},
        "stage_ms": {k: round(st[k], 3) for k in ("upload_ms", "detect_ms", "describe_ms", "d2h_ms", "total_ms")},
        "files_stage_ms": {k: round(st_files[k], 3) for k in ("describe_ms", "d2h_ms", "write_ms", "total_ms")},
        "describe_hidden_ms": round(hidden, 3),
        "describe_hidden_share": hidden / st["describe_ms"] if st["describe_ms"] else None,
        "cpu_reference_s_per_image": cpu_s / min(a.parity, n) if a.parity else None, "parity": bool(parity),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--parity", type=int, default=2)
    ap.add_argument("--threshold", type=float, default=1e-3)
    ap.add_argument("--out-dir", default=None, help="where the files arm writes (default: a temporary directory)")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    out_root = a.out_dir or tempfile.mkdtemp(prefix="r3d_features_")
    ctx = capi.Context((0,))
    try:
        res = [run_workload(ctx, n, w, h, a, out_root) for n, w, h in WORKLOADS]
    finally:
        ctx.close()
        if a.out_dir is None:
            shutil.rmtree(out_root, ignore_errors=True)
    parity = all(r["parity"] for r in res)
    print(json.dumps({"workload": "extract_features", "gpu": gpu[0] if gpu else "unknown", "results": res,
                      "parity": parity}))
    return 0 if parity else 1


if __name__ == "__main__":
    sys.exit(main())
