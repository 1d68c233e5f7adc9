#!/usr/bin/env python
"""Small-shape pass over every kernel family for `compute-sanitizer` (memcheck / racecheck / synccheck / initcheck):

    compute-sanitizer --tool racecheck python scripts/sanitize_small.py [match|filter|ba|liop|cascade|ba_envelope|chol|all]

Shapes are tiny on purpose (the sanitizer serialises everything); correctness of the results is checked by the
`-m gpu` tests, this script only has to execute every kernel once."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np

from regard3d_b200 import capi, synth

what = sys.argv[1] if len(sys.argv) > 1 else "all"
ctx = capi.Context((0,))
n_feats = int(os.environ.get("SAN_FEATS", "600"))
if what in ("match", "filter", "all"):
    sc = synth.make_scene(3, n_feats, 144, "liop", seed=5)
    pairs = synth.exhaustive_pairs(3)
    for v in range(3):
        ctx.upload_regions(v, sc["descs"][v], sc["xys"][v])
    m = ctx.match_pairs(pairs, 0.6)
    print("match f32/144:", m.total, "matches", ctx.match_timing()["kernel_launches"], "launches")
    if what in ("match", "all"):
        idx, dist = ctx.search_neighbours(0, 1, n_feats)
        ctx.clear_regions()
        s8 = synth.make_scene(3, n_feats, 128, "sift", seed=6, as_u8=True)
        for v in range(3):
            ctx.upload_regions(v, s8["descs"][v], s8["xys"][v])
        m8 = ctx.match_pairs(pairs, 0.6)
        print("match u8/128:", m8.total, "matches")
        m8 = ctx.match_pairs(pairs, 0.6, capi.MATCH_EXACT_SCAN)
        print("exact scan u8/128:", m8.total, "matches")
        ctx.clear_regions()
        for v in range(3):
            ctx.upload_regions(v, sc["descs"][v], sc["xys"][v])
    if what in ("filter", "all"):
        for model in (capi.MODEL_F, capi.MODEL_H, capi.MODEL_E):
            f = ctx.filter_pairs(m, sc["widths"], sc["heights"], model=model, max_iter=int(os.environ.get("SAN_ITERS", "256")))
            print("filter model", model, ":", f.total, "inliers")
if what in ("ba", "all"):
    prob = synth.make_ba_problem(n_cams=8, n_pts=400, obs_per_pt=4, seed=2)
    arrs = {}
    for k in ("poses", "intrinsics", "points", "obs_xy"):
        arrs[k] = np.ascontiguousarray(prob[k], np.float64)
    for k in ("obs_cam", "obs_pt", "cam_intr"):
        arrs[k] = np.ascontiguousarray(prob[k], np.uint32)
    s, trace = ctx.bundle_adjust(arrs, max_iterations=3)
    print("ba:", s["iterations"], "iterations, cost", trace[0], "->", trace[-1])
    ctx.ba_residuals(arrs)
    # the CTA-per-point Schur kernel and the points no Schur kernel visits: point 0 gets a 36-observation track (every
    # camera, camera 0 five times), one more point has no observation at all
    extra = np.concatenate([np.arange(8), np.zeros(28, int)]).astype(np.uint32)
    arrs["obs_cam"] = np.concatenate([arrs["obs_cam"], extra])
    arrs["obs_pt"] = np.concatenate([arrs["obs_pt"], np.zeros(len(extra), np.uint32)])
    arrs["obs_xy"] = np.concatenate([arrs["obs_xy"], arrs["obs_xy"][:1] + np.linspace(-1.0, 1.0, len(extra))[:, None]])
    arrs["points"] = np.concatenate([arrs["points"], arrs["points"][:1] + 1.0])
    s, trace = ctx.bundle_adjust(arrs, max_iterations=3)
    print("ba (long track, repeated camera, unobserved point):", s["iterations"], "iterations, cost", trace[0], "->", trace[-1])
    step = ctx.debug_ba_step(arrs, 1e4)
    print("ba step: %d batches, %d CTA points, |delta| %.3g" % (step["n_batches"], step["n_long"], np.linalg.norm(step["delta"])))
if what in ("cascade", "all"):
    s8 = synth.make_scene(3, n_feats, 128, "sift", seed=6, as_u8=True)
    ctx.clear_regions()
    for v in range(3):
        ctx.upload_regions(v, s8["descs"][v], s8["xys"][v])
    mc = ctx.match_pairs(synth.exhaustive_pairs(3), 0.8, capi.MATCH_CASCADE_HASHING)
    print("cascade u8/128:", mc.total, "matches")
    sf = synth.make_scene(3, n_feats, 144, "liop", seed=7)
    ctx.clear_regions()
    for v in range(3):
        ctx.upload_regions(v, sf["descs"][v], sf["xys"][v])
    mc = ctx.match_pairs(synth.exhaustive_pairs(3), 0.8, capi.MATCH_CASCADE_HASHING)
    print("cascade f32/144:", mc.total, "matches")
if what in ("ba_envelope", "all"):
    os.environ["R3D_BA_CHOL"] = "envelope"
    prob = synth.make_ba_problem(n_cams=37, n_pts=1500, obs_per_pt=4, seed=41)
    arrs = {}
    for k in ("poses", "intrinsics", "points", "obs_xy"):
        arrs[k] = np.ascontiguousarray(prob[k], np.float64)
    for k in ("obs_cam", "obs_pt", "cam_intr"):
        arrs[k] = np.ascontiguousarray(prob[k], np.uint32)
    s, trace = ctx.bundle_adjust(arrs, max_iterations=2)
    print("ba (envelope Cholesky, cluster of 8):", s["iterations"], "iterations, cost", trace[0], "->", trace[-1])
    del os.environ["R3D_BA_CHOL"]
if what in ("chol", "all"):
    # the dense solvers through their debug entry points: k_chol_fused at n = 33 (a partial second panel, rhs row in
    # the last diagonal tile), k_chol_envelope at n = 64 on a cluster of 2 (rhs row in a tile of its own), and
    # k_chol_fused + k_rotavg_trsm3 on 33 x 3 right-hand sides
    rng = np.random.default_rng(3)
    for n, method, ft, grid in ((33, capi.CHOL_DENSE, None, 0), (64, capi.CHOL_ENVELOPE, np.array([0, 0, 0], np.int32), 2)):
        G = rng.standard_normal((n, n))
        A = np.vstack([G @ G.T + n * np.eye(n), rng.standard_normal((1, n))])
        L, x, _, bad = ctx.debug_cholesky(A, method, ft=ft, grid=grid)
        print("chol method %d n %d: residual %.2e, not_pd %d" % (method, n, np.abs(A[:n] @ x - A[n]).max(), bad))
    G = rng.standard_normal((33, 33))
    A = G @ G.T + 33 * np.eye(33)
    Y = rng.standard_normal((33, 3))
    X = ctx.debug_chol_solve3(A, Y)
    print("chol_solve3 n 33: residual %.2e" % np.abs(A @ X - Y).max())
if what in ("liop", "all"):
    rng = np.random.default_rng(1)
    img = rng.random((120, 160)).astype(np.float32)
    kps = np.stack([rng.uniform(-5, 165, 40), rng.uniform(-5, 125, 40), rng.uniform(3, 30, 40), rng.uniform(0, 360, 40)], 1)
    d = ctx.liop_describe(img, kps.astype(np.float32), 8.0)
    print("liop:", d.shape, float(np.linalg.norm(d, axis=1).mean()))
ctx.close()
print("sanitize_small: done")
