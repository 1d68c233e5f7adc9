"""-m gpu: r3d_resect_views against the CPU oracle (orc_resect_views): the same status, inlier sequence, errorMax and
AC-RANSAC pose bit for bit; with the pose refinement the same LM iteration / accept sequence and the final cost within
1e-8 relative (the bars of test_gpu_relpose.py)."""
import numpy as np
import pytest

from oracle import pyoracle_resection as pro
from regard3d_b200 import synth
from resection_scenes import make_batch, make_view, rotation_angle_deg

pytestmark = pytest.mark.gpu


def _flat(views):
    counts = [len(v["X"]) for v in views]
    X = np.concatenate([v["X"] for v in views]) if sum(counts) else np.zeros((0, 3))
    x = np.concatenate([v["x"] for v in views]) if sum(counts) else np.zeros((0, 2))
    return counts, X, x


def _run(ctx, r3dlib, views, **opts):
    counts, X, x = _flat(views)
    rv = r3dlib.resection_views(counts, [v["width"] for v in views], [v["height"] for v in views], [v["model"] for v in views],
                                [v["focal"] for v in views], [v["ppx"] for v in views], [v["ppy"] for v in views],
                                [v["disto"] for v in views])
    got, gofs, ginl = ctx.resect_views(rv, X, x, **opts)
    first = np.concatenate([[0], np.cumsum(counts)[:-1]]) if counts else []
    intrs = np.array([pro.intr8(v["focal"], v["ppx"], v["ppy"], v["disto"]) for v in views])
    exp, eofs, einl = pro.resect_views(first, counts, [v["width"] for v in views], [v["height"] for v in views],
                                       [v["model"] for v in views], intrs, X, x, **opts)
    refine = opts.get("refine", True)
    assert len(got) == len(exp) == len(views)
    for a, (g, e, v) in enumerate(zip(got, exp, views)):
        assert g["status"] == e["status"], (a, g["status"], e["status"])
        gi, ei = ginl[int(gofs[a]):int(gofs[a + 1])], einl[int(eofs[a]):int(eofs[a + 1])]
        assert np.array_equal(gi, ei), "view %d: inlier sequence differs" % a
        if e["status"] != pro.RESECT_OK:
            assert g["n_inliers"] == 0 and g["lm_termination"] == -1
            continue
        for f in ("n_inliers", "found_residual_precision", "rotation_ransac", "translation_ransac"):
            assert np.array_equal(g[f], e[f]), (a, f)
        if not refine:
            assert g["lm_termination"] == -1 and np.array_equal(g["rotation"], e["rotation_ransac"])
            assert np.array_equal(g["translation"], e["translation_ransac"]) and np.array_equal(g["center"], e["center"])
            continue
        for f in ("lm_iterations", "lm_successful_steps", "lm_termination"):
            assert g[f] == e[f], (a, f, g[f], e[f])
        assert abs(g["lm_final_cost"] - e["lm_final_cost"]) <= 1e-8 * e["lm_final_cost"] + 1e-18, a
        sc = max(1.0, v["scale"])
        assert np.allclose(g["rotation"], e["rotation"], atol=1e-7), a
        assert np.allclose(g["translation"], e["translation"], atol=1e-6 * sc), a
        assert np.allclose(g["center"], e["center"], atol=1e-6 * sc), a
    return got, exp


def _same(a, b):
    """Every field bit for bit (the records' padding bytes are not part of the result)."""
    return all(np.array_equal(a[f], b[f]) for f in a.dtype.names)


def _close_to_truth(got, views, deg=0.1, rel=1e-3):
    for g, v in zip(got, views):
        assert g["status"] == 0
        assert rotation_angle_deg(g["rotation"], v["R"]) < deg
        assert np.abs(g["center"] - v["C"]).max() < rel * v["scale"]


def test_clean_batch_of_40_views(gpu_ctx, r3dlib):
    views = make_batch(1, 40, 600, outliers=0.0)
    got, _ = _run(gpu_ctx, r3dlib, views)
    _close_to_truth(got, views)
    t = gpu_ctx.resection_timing()
    assert t["kernel_launches"] >= 4 and t["lm_iterations"] > 0


def test_forty_percent_outliers(gpu_ctx, r3dlib):
    views = make_batch(2, 12, 1500, outliers=0.4)
    got, _ = _run(gpu_ctx, r3dlib, views)
    _close_to_truth(got, views)
    for g, v in zip(got, views):
        assert g["n_inliers"] >= 0.95 * v["inlier"].sum()


def test_four_to_nine_correspondences_and_too_few(gpu_ctx, r3dlib):
    views = [make_view(300 + m, m, noise=0.1) for m in (0, 1, 3, 4, 5, 6, 7, 8, 9)]
    got, _ = _run(gpu_ctx, r3dlib, views)
    assert [int(s) for s in got["status"][:3]] == [r3dlib.RESECT_TOO_FEW] * 3
    assert all(int(s) != r3dlib.RESECT_TOO_FEW for s in got["status"][3:])


def test_no_intrinsic(gpu_ctx, r3dlib):
    views = make_batch(4, 3, 200)
    views[1]["focal"] = 0.0
    got, _ = _run(gpu_ctx, r3dlib, views)
    assert [int(s) for s in got["status"]] == [0, r3dlib.RESECT_NO_INTRINSIC, 0]


@pytest.mark.parametrize("model", [1, 2, 3, 4, 5])
def test_camera_models_with_distortion(gpu_ctx, r3dlib, model):
    views = make_batch(50 + model, 4, 800, models=(model,), outliers=0.2)
    got, _ = _run(gpu_ctx, r3dlib, views)
    _close_to_truth(got, views)


def test_huge_view(gpu_ctx, r3dlib):
    views = [make_view(6, 20000, outliers=0.3), make_view(7, 300)]
    got, _ = _run(gpu_ctx, r3dlib, views, max_iter=256)
    _close_to_truth(got, views)


def test_finite_precision_and_tiny_budget(gpu_ctx, r3dlib):
    views = make_batch(8, 6, 500, outliers=0.3)
    _run(gpu_ctx, r3dlib, views, precision_px=4.0)
    _run(gpu_ctx, r3dlib, views, precision_px=0.05)
    _run(gpu_ctx, r3dlib, views, max_iter=3)
    _run(gpu_ctx, r3dlib, views, max_iter=15, precision_px=2.0)


def test_all_outliers_is_no_model(gpu_ctx, r3dlib):
    v = make_view(9, 400, outliers=1.0)
    got, _ = _run(gpu_ctx, r3dlib, [v], max_iter=512)
    assert got["status"][0] == r3dlib.RESECT_NO_MODEL


def test_mixed_batch_without_refinement_and_repeat(gpu_ctx, r3dlib):
    views = [make_view(400 + k, m, model=md, outliers=o) for k, (m, md, o) in enumerate(
        [(3000, 3, 0.3), (2, 1, 0.0), (50, 5, 0.1), (1200, 4, 0.5), (9000, 2, 0.2), (700, 1, 1.0), (17000, 3, 0.2)])]
    views[2]["focal"] = -1.0
    a, _ = _run(gpu_ctx, r3dlib, views, refine=False, max_iter=512)
    b, _ = _run(gpu_ctx, r3dlib, views, max_iter=512)
    c, _ = _run(gpu_ctx, r3dlib, views, max_iter=512)
    assert _same(b, c)
    assert np.array_equal(a["rotation_ransac"], b["rotation_ransac"])


def test_two_devices_equal_one(r3dlib):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    views = make_batch(10, 16, 900, outliers=0.3)
    c1, c2 = r3dlib.Context((0,)), r3dlib.Context((0, 1))
    a, _ = _run(c1, r3dlib, views)
    b, _ = _run(c2, r3dlib, views)
    assert _same(a, b)
    c1.close()
    c2.close()


def test_invalid_input(gpu_ctx, r3dlib):
    views = make_batch(11, 2, 100)

    def call(vs, **opts):
        counts, X, x = _flat(vs)
        rv = r3dlib.resection_views(counts, [v["width"] for v in vs], [v["height"] for v in vs], [v["model"] for v in vs],
                                    [v["focal"] for v in vs], [v["ppx"] for v in vs], [v["ppy"] for v in vs],
                                    [v["disto"] for v in vs])
        return gpu_ctx.resect_views(rv, X, x, **opts)

    def bad(**change):
        vs = [dict(v) for v in views]
        for k, val in change.items():
            vs[1][k] = val
        return vs

    nanX, infx = views[1]["X"].copy(), views[1]["x"].copy()
    nanX[5, 1] = np.nan
    infx[7, 0] = np.inf
    cases = [(bad(X=nanX), {}), (bad(x=infx), {}), (bad(model=9), {}), (bad(width=0), {}), (views, dict(refine_intrinsics=1)),
             (views, dict(max_iter=0)), (views, dict(precision_px=-1.0)), (bad(disto=(np.nan, 0, 0)), {})]
    for vs, opts in cases:
        with pytest.raises(r3dlib.R3DError) as e:
            call(vs, **opts)
        assert e.value.code == -1
    sd = r3dlib.SfmData()
    sd.add_intrinsic(0, r3dlib.CAM_PINHOLE, 100, 100, 110.0, 50.0, 50.0)
    sd.add_view(0, "a.jpg", 100, 100, id_intrinsic=0, id_pose=0)
    sd.add_view(1, "b.jpg", 100, 100, id_intrinsic=7, id_pose=1)
    sd.add_pose(0, np.eye(3), np.zeros(3))
    for ids in ([0], [5], [1]):  # already has a pose, unknown view, unknown intrinsic
        with pytest.raises(r3dlib.R3DError) as e:
            gpu_ctx.sfm_resect_views(sd, ids)
        assert e.value.code == -1


def test_end_to_end_bring_back_two_views_of_the_ring(gpu_ctx, r3dlib):
    """The global chain of test_gpu_transavg's end-to-end test on its 8-view ring, bundle-adjusted; then two views lose
    their poses, sfm_resect_views(every view without a pose) brings them back from the structure, and a bundle
    adjustment over all views follows."""
    n = 8
    sc = synth.make_scene(n, 1500, 64, "msurf", seed=61)
    pairs = synth.exhaustive_pairs(n)
    gpu_ctx.clear_regions()
    for v in range(n):
        gpu_ctx.upload_regions(v, sc["descs"][v], sc["xys"][v])
    put = gpu_ctx.match_pairs(pairs, 0.8)
    Ks = np.array([[1.1 * max(int(w), int(h)), w / 2.0, h / 2.0] for w, h in zip(sc["widths"], sc["heights"])])
    rel, inl = gpu_ctx.relative_poses(put, sc["widths"], sc["heights"], Ks)
    Rg, rk, ek_rot, _, _ = gpu_ctx.rotation_averaging(rel, n)
    C, _, vk, _, S = gpu_ctx.translation_averaging(rel, Rg, rk, n, edge_use=ek_rot)
    assert S["success"] and vk.all()

    def new_sd(poses):
        sd = r3dlib.SfmData()
        sd.add_intrinsic(0, r3dlib.CAM_PINHOLE, sc["w"], sc["h"], Ks[0][0], Ks[0][1], Ks[0][2])
        for v in range(n):
            sd.add_view(v, "image%06d.jpg" % v, sc["w"], sc["h"], id_intrinsic=0, id_pose=v)
        for v, (R, c) in poses.items():
            sd.add_pose(v, R, c)
        return sd

    sd = new_sd({v: (Rg[v], C[v]) for v in range(n)})
    gpu_ctx.structure_from_tracks(sd, r3dlib.Tracks.build(inl, 2))
    gpu_ctx.remove_outliers(sd, 4.0, 2, 2.0)
    gpu_ctx.sfm_bundle_adjust(sd, max_iterations=50, refine_intrinsics=0)
    ba = {p["id"]: (p["R"], p["center"]) for p in sd.poses()}
    lost = (2, 5)
    sd2 = new_sd({v: ba[v] for v in range(n) if v not in lost})
    for lm in sd.landmarks():
        sd2.add_landmark(lm["id"], lm["X"], lm["obs"])
    got = gpu_ctx.sfm_resect_views(sd2)
    assert [int(g["view_id"]) for g in got] == list(lost) and (got["status"] == 0).all()
    back = {p["id"]: (p["R"], p["center"]) for p in sd2.poses()}
    cs = np.array([ba[v][1] for v in range(n)])
    diameter = np.linalg.norm(cs[:, None] - cs[None], axis=2).max()
    for g in got:
        v = int(g["view_id"])
        assert np.array_equal(back[v][0], g["rotation"]) and np.array_equal(back[v][1], g["center"])
        assert np.linalg.norm(back[v][1] - ba[v][1]) <= 2e-3 * diameter
        assert rotation_angle_deg(back[v][0], ba[v][0]) <= 0.1
    s = gpu_ctx.sfm_bundle_adjust(sd2, max_iterations=50)
    rms = np.sqrt(2.0 * s["final_cost"] / max(1, sum(len(lm["obs"]) for lm in sd2.landmarks())))
    print("resected views %s: %s inliers, RMS after BA %.3f px" % (lost, got["n_inliers"].tolist(), rms))
    assert rms < 0.8
