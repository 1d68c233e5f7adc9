"""-m gpu: the steps either side of bundle adjustment (SURVEY.md 8f-3) through the C ABI: matches -> tracks -> landmarks
triangulated from known poses -> outlier rejection -> bundle adjustment, i.e. the BA kernel reached from `matches.f`
without OpenMVG (what SfM_Data_Structure_Computation_Blind + sfm_data_filters + Bundle_Adjustment_Ceres do upstream)."""
import numpy as np
import pytest

from regard3d_b200 import synth

pytestmark = pytest.mark.gpu


def _scene_sfm(r3dlib, sc, pose_noise=0.0, seed=0):
    rng = np.random.default_rng(seed)
    n = len(sc["descs"])
    sd = r3dlib.SfmData()
    sd.add_intrinsic(0, r3dlib.CAM_RADIAL3, sc["w"], sc["h"], sc["f"], sc["w"] / 2.0, sc["h"] / 2.0, (0.0, 0.0, 0.0))
    for v in range(n):
        sd.add_view(v, "image%06d.jpg" % v, sc["w"], sc["h"], id_intrinsic=0, id_pose=v)
        R = synth._rodrigues(sc["poses"][v, :3] + pose_noise * rng.standard_normal(3))
        t = sc["poses"][v, 3:] + pose_noise * rng.standard_normal(3)
        sd.add_pose(v, R, -R.T @ t)
    return sd


def _flat(sd):
    """The landmarks of an SfmData as the oracle's flat arrays (cameras = poses in id order, one intrinsic group)."""
    poses = []
    for p in sd.poses():
        R, C = p["R"], p["center"]
        poses.append(np.concatenate([synth._log_so3(R), -R @ C]))
    intr = np.array([[i["focal"], i["ppx"], i["ppy"]] + i["disto"][:3] for i in sd.intrinsics()])
    lms = sd.landmarks()
    ofs, cam, xy, X = [0], [], [], []
    for lm in lms:
        for (v, f, x, y) in lm["obs"]:
            cam.append(v); xy.append((x, y))
        ofs.append(len(cam)); X.append(lm["X"])
    return (np.array(poses), intr, np.array(ofs, np.uint64), np.array(cam, np.uint32), np.array(xy, np.float64).reshape(-1, 2),
            np.array(X, np.float64).reshape(-1, 3), lms)


def test_matches_to_tracks_to_structure_to_ba(gpu_ctx, oracle, r3dlib):
    sc = synth.make_scene(6, 1500, 64, "msurf", seed=61)
    pairs = synth.exhaustive_pairs(6)
    gpu_ctx.clear_regions()
    for v in range(6):
        gpu_ctx.upload_regions(v, sc["descs"][v], sc["xys"][v])
    put = gpu_ctx.match_pairs(pairs, 0.7)
    geo = gpu_ctx.filter_pairs(put, sc["widths"], sc["heights"])
    tracks = r3dlib.Tracks.build(geo, 2)
    assert len(tracks) > 300
    sd = _scene_sfm(r3dlib, sc)
    rejected = gpu_ctx.structure_from_tracks(sd, tracks)
    poses, intr, ofs, cam, xy, X, lms = _flat(sd)
    assert len(lms) + rejected == len(tracks) and len(lms) > 300
    # every kept landmark: the oracle triangulates the same point from the same observations
    Xo, ok = oracle.triangulate_landmarks(ofs, cam, xy, poses, np.zeros(6, np.uint32), intr)
    assert ok.all()
    assert np.abs(X - Xo).max() <= 1e-7 * max(1.0, np.abs(Xo).max())
    # ground truth: tracks of true correspondences land on their 3-D point
    err = []
    for lm in lms:
        tids = {int(sc["truth"][v][f]) for (v, f, _, _) in lm["obs"]}
        if len(tids) == 1 and -1 not in tids:
            err.append(np.linalg.norm(np.array(lm["X"]) - sc["points"][tids.pop()]))
    assert len(err) > 250 and np.median(err) < 0.05
    # outlier rejection: the observations kept and the angle decisions equal the oracle's, then BA on what is left
    keep_o, ang_o = oracle.landmark_checks(ofs, cam, xy, poses, np.zeros(6, np.uint32), intr, X, 4.0)
    # the angle test runs on what the residual test left: the oracle's largest angle over the kept observations
    kofs = np.r_[0, np.cumsum(np.add.reduceat(keep_o.astype(np.int64), ofs[:-1].astype(np.int64)))].astype(np.uint64)
    _, ang_kept = oracle.landmark_checks(kofs, cam[keep_o], xy[keep_o], poses, np.zeros(6, np.uint32), intr, X, np.inf)
    n_obs_before = sum(len(lm["obs"]) for lm in lms)
    rm_obs, rm_lm = gpu_ctx.remove_outliers(sd, 4.0, 2, 2.0)
    assert rm_obs == int((~keep_o).sum())
    expected = {}
    for l, lm in enumerate(lms):
        k = keep_o[int(ofs[l]):int(ofs[l + 1])]
        kept = sorted((v, f) for (v, f, _, _), kk in zip(lm["obs"], k) if kk)
        assert ang_kept[l] <= ang_o[l] + 1e-12
        if len(kept) >= 2 and ang_kept[l] >= 2.0:
            expected[lm["id"]] = kept
    after = sd.landmarks()
    assert {lm["id"]: sorted((v, f) for (v, f, _, _) in lm["obs"]) for lm in after} == expected
    assert sum(len(lm["obs"]) for lm in after) == n_obs_before - rm_obs and len(after) == len(lms) - rm_lm
    s = gpu_ctx.sfm_bundle_adjust(sd, max_iterations=25)
    assert s["final_cost"] <= s["initial_cost"] and s["iterations"] >= 1
    res = np.sqrt(2.0 * s["final_cost"] / max(1, sum(len(lm["obs"]) for lm in after)))
    assert res < 1.5                                         # RMS reprojection error in pixels (0.5 px feature noise)


def test_triangulation_rejects_points_behind_a_camera(gpu_ctx, r3dlib):
    sc = synth.make_scene(3, 400, 32, "msurf", seed=62)
    gpu_ctx.clear_regions()
    for v in range(3):
        xy = sc["xys"][v].copy()
        gpu_ctx.upload_regions(v, sc["descs"][v], xy)
    sd = _scene_sfm(r3dlib, sc)
    # a "track" made of unrelated features triangulates behind a camera or far off: it must not survive both steps
    pairs = np.array([[0, 1]], np.uint32)
    m = np.array([(k, (k * 7 + 3) % 400) for k in range(60)], r3dlib.indmatch_dtype)
    tr = r3dlib.Tracks.build(r3dlib.Matches.from_csr(pairs, np.array([0, 60], np.uint64), m), 2)
    rejected = gpu_ctx.structure_from_tracks(sd, tr)
    rm_obs, rm_lm = gpu_ctx.remove_outliers(sd, 4.0, 2, 2.0)
    assert rejected + rm_lm >= 50 and len(sd.landmarks()) <= 10
