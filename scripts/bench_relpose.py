"""Relative poses of every E-filtered pair (r3d_relative_poses) on one GPU, against the CPU restatement.

    python scripts/bench_relpose.py [--images 60] [--feats 10000] [--steps 5] [--warmup 1] [--sample 24]

Scene: a seeded ring scene (synth.make_scene, SIFT-like uint8 descriptors).  Putative matching and the essential filter
run once; the timed region is r3d_relative_poses on the E-filtered pairs, ending in a device synchronise (the call
returns host results).  The CPU arm is orc_relative_poses (OpenMP over pairs, all usable CPUs, as upstream's loop) on
a seeded sample of the pairs; parity_on_sample compares the two on that sample.  Prints one JSON line.  Writes nothing.
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
    ap.add_argument("--images", type=int, default=60)
    ap.add_argument("--feats", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=24)
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    from regard3d_b200 import build, capi, synth
    from oracle import pyoracle as po
    from oracle import pyoracle_relpose as por
    build.build()
    sc = synth.make_scene(a.images, a.feats, 128, "sift", seed=a.seed, as_u8=True)
    pairs = synth.exhaustive_pairs(a.images)
    Ks = np.array([[1.1 * max(int(w), int(h)), w / 2.0, h / 2.0] for w, h in zip(sc["widths"], sc["heights"])])
    ctx = capi.Context((0,))
    for v in range(a.images):
        ctx.upload_regions(v, sc["descs"][v], sc["xys"][v])
    put = ctx.match_pairs(pairs, 0.8)
    ef = ctx.filter_pairs(put, sc["widths"], sc["heights"], model=capi.MODEL_E, Ks=Ks)
    for _ in range(a.warmup):
        ctx.relative_poses(ef, sc["widths"], sc["heights"], Ks)
    times = []
    for _ in range(a.steps):
        t0 = time.perf_counter()
        got, _ = ctx.relative_poses(ef, sc["widths"], sc["heights"], Ks)
        times.append(time.perf_counter() - t0)
    timing = ctx.relpose_timing()
    n_pairs = len(got)
    # CPU arm on a seeded sample of the E-filtered pairs
    e_pairs, e_ofs, e_m = ef.export_csr()
    rng = np.random.default_rng(a.seed)
    sel = np.sort(rng.choice(n_pairs, min(a.sample, n_pairs), replace=False))
    s_ofs = np.zeros(len(sel) + 1, np.uint64)
    chunks = []
    for k, p in enumerate(sel):
        chunks.append(e_m[int(e_ofs[p]):int(e_ofs[p + 1])])
        s_ofs[k + 1] = s_ofs[k] + len(chunks[-1])
    n_thr = len(os.sched_getaffinity(0))
    t0 = time.perf_counter()
    exp, _, _ = por.relative_poses(sc["xys"], sc["widths"], sc["heights"], Ks, e_pairs[sel], s_ofs, np.concatenate(chunks),
                                  n_threads=n_thr)
    cpu_s = time.perf_counter() - t0
    parity = True
    for g, e in zip(got[sel], exp):
        parity &= bool(g["status"] == e["status"] and np.array_equal(g["E"], e["E"]) and g["n_inliers"] == e["n_inliers"])
        if e["status"] == por.RELPOSE_OK:
            parity &= bool(g["ba_iterations"] == e["ba_iterations"] and g["ba_termination"] == e["ba_termination"]
                           and abs(g["ba_final_cost"] - e["ba_final_cost"]) <= 1e-8 * e["ba_final_cost"])
    med = float(np.median(times))
    res = {"metric": "relpose_pairs_per_s", "images": a.images, "feats": a.feats, "pairs": n_pairs,
           "ok_pairs": int((got["status"] == 0).sum()), "matches": int(ef.total),
           "gpu_pairs_per_s": n_pairs / med, "gpu_s_median": med, "gpu_s_all": times, "relpose_timing": timing,
           "cpu_pairs_per_s": len(sel) / cpu_s, "cpu_threads": n_thr, "cpu_sample_pairs": int(len(sel)),
           "parity_on_sample": parity, "ba_iterations_mean": float(got["ba_iterations"].mean())}
    res.update(gpu_info())
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
