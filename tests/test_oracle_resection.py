"""The CPU oracle of the resection step (oracle/oracle_resection.cpp) pinned by independent means: the truth of synthetic
scenes, the constraints a P3P solution satisfies, numpy restatements of the camera models, OpenCV where it is
installed, and scipy's minimiser on the refinement's cost."""
import numpy as np
import pytest

from oracle import pyoracle as po
from oracle import pyoracle_resection as pro
from resection_scenes import DISTO, distort, make_view, project, rodrigues, rotation_angle_deg


def _K(v):
    return np.array([[v["focal"], 0, v["ppx"]], [0, v["focal"], v["ppy"]], [0, 0, 1.0]])


def _poses(v, P):
    Ki = np.linalg.inv(_K(v))
    return [(Ki @ p[:, :3], Ki @ p[:, 3]) for p in P]


def test_p3p_contains_the_truth_and_satisfies_its_constraints():
    n_models = 0
    for seed in range(200):
        v = make_view(seed, 3, model=1, noise=0.0)
        P = pro.p3p([v["focal"], v["ppx"], v["ppy"]], v["X"], v["x"])
        assert 1 <= len(P) <= 4
        n_models += len(P)
        Pt = _K(v) @ np.c_[v["R"], v["t"]]
        assert min(np.abs(p - Pt).max() for p in P) <= 1e-9 * np.abs(Pt).max(), seed
        for R, t in _poses(v, P):
            assert np.abs(R @ R.T - np.eye(3)).max() <= 1e-9 and abs(np.linalg.det(R) - 1.0) <= 1e-9
            Y = v["X"] @ R.T + t  # the three points in the camera frame: on their bearings, same mutual distances
            assert (Y[:, 2] > 0).all()
            px = Y[:, :2] / Y[:, 2:] * v["focal"] + [v["ppx"], v["ppy"]]
            assert np.abs(px - v["x"]).max() <= 1e-6
            for i, j in ((0, 1), (0, 2), (1, 2)):
                d = np.linalg.norm(v["X"][i] - v["X"][j])
                assert abs(np.linalg.norm(Y[i] - Y[j]) - d) <= 1e-9 * d
    assert n_models > 250  # samples with more than one real solution occur


def test_p3p_solution_set_equals_opencv():
    cv2 = pytest.importorskip("cv2")
    for seed in range(40):
        v = make_view(1000 + seed, 3, model=1, noise=0.0)
        mine = _poses(v, pro.p3p([v["focal"], v["ppx"], v["ppy"]], v["X"], v["x"]))
        n, rv, tv = cv2.solveP3P(v["X"], v["x"], _K(v), None, flags=cv2.SOLVEPNP_P3P)
        theirs = [(cv2.Rodrigues(r)[0], t.ravel()) for r, t in zip(rv, tv)]
        theirs = [(R, t) for R, t in theirs if ((v["X"] @ R.T + t)[:, 2] > 0).all()]
        assert len(mine) == len(theirs), seed
        for R, t in theirs:
            assert min(max(np.abs(R - Rm).max(), np.abs(t - tm).max() / max(1.0, np.abs(t).max())) for Rm, tm in mine) <= 1e-6


def test_p3p_degenerate_samples_give_no_model():
    v = make_view(5, 3, model=1, noise=0.0)
    K = [v["focal"], v["ppx"], v["ppy"]]
    line = np.array([v["X"][0], v["X"][0] + (v["X"][1] - v["X"][0]) * 0.5, v["X"][1]])
    twice = np.array([v["X"][0], v["X"][0], v["X"][2]])
    for X in (line, twice, np.zeros((3, 3))):
        assert len(pro.p3p(K, X, v["x"])) == 0
    same_pixel = np.array([v["x"][0], v["x"][0], v["x"][0]])
    P = pro.p3p(K, v["X"], same_pixel)
    assert np.isfinite(P).all()


@pytest.mark.parametrize("model", [1, 2, 3, 4, 5])
def test_undistortion_inverts_the_camera_model(model):
    v = make_view(20 + model, 2000, model=model, noise=0.0)
    intr = pro.intr8(v["focal"], v["ppx"], v["ppy"], v["disto"])
    xu = pro.undistort(model, intr, v["x"])
    xd, yd = distort(model, v["disto"], (xu[:, 0] - v["ppx"]) / v["focal"], (xu[:, 1] - v["ppy"]) / v["focal"])
    back = np.stack([v["ppx"] + v["focal"] * xd, v["ppy"] + v["focal"] * yd], 1)
    assert np.abs(back - v["x"]).max() <= 1e-9
    if model > 1:
        assert np.abs(xu - v["x"]).max() > 1.0  # the distortion of these scenes is not negligible
    # the numpy camera model of the scenes is the oracle's residual functor
    for k in range(0, 2000, 400):
        r, _ = po.ba_jacobian_model(model, intr[:6], intr[6:], np.zeros(6), [(xu[k, 0] - v["ppx"]) / v["focal"],
                                                                             (xu[k, 1] - v["ppy"]) / v["focal"], 1.0], np.zeros(2))
        assert np.abs(r - v["x"][k]).max() <= 1e-9


@pytest.mark.parametrize("model", [1, 3, 5])
def test_acransac_finds_the_pose_under_outliers(model):
    v = make_view(40 + model, 1500, model=model, outliers=0.3)
    intr = pro.intr8(v["focal"], v["ppx"], v["ppy"], v["disto"])
    r, inl = pro.resect_view(v["X"], v["x"], v["width"], v["height"], model, intr)
    assert r["status"] == pro.RESECT_OK and r["n_inliers"] == len(inl) == len(set(inl.tolist()))
    for R, C in ((r["rotation_ransac"], -r["rotation_ransac"].T @ r["translation_ransac"]), (r["rotation"], r["center"])):
        assert rotation_angle_deg(R, v["R"]) <= 0.1
        assert np.abs(C - v["C"]).max() <= 1e-3 * v["scale"]
    assert np.isin(np.nonzero(v["inlier"])[0], inl).mean() >= 0.95
    assert r["lm_termination"] in (1, 2, 3) and r["lm_final_cost"] <= r["lm_initial_cost"]
    assert 0.0 < r["found_residual_precision"] < 3.0
    # residuals of the listed inliers come in ascending order and end at the reported precision
    xu = pro.undistort(model, intr, v["x"])
    pr = v["X"] @ r["rotation_ransac"].T + r["translation_ransac"]
    e = np.linalg.norm(pr[:, :2] / pr[:, 2:] * v["focal"] + [v["ppx"], v["ppy"]] - xu, axis=1)[inl]
    assert (np.diff(e) >= -1e-9).all() and abs(e[-1] - r["found_residual_precision"]) <= 1e-9


def test_acransac_overlaps_opencv_ransac():
    cv2 = pytest.importorskip("cv2")
    v = make_view(77, 1000, model=1, outliers=0.3)
    r, inl = pro.resect_view(v["X"], v["x"], v["width"], v["height"], 1, pro.intr8(v["focal"], v["ppx"], v["ppy"]))
    ok, _, _, cv_inl = cv2.solvePnPRansac(v["X"], v["x"], _K(v), None, reprojectionError=2.0, iterationsCount=2000)
    assert ok
    cv_inl = cv_inl.ravel()
    assert np.isin(cv_inl, inl).mean() >= 0.9


def test_statuses():
    v = make_view(3, 400, outliers=1.0)
    intr = pro.intr8(v["focal"], v["ppx"], v["ppy"], v["disto"])
    assert pro.resect_view(v["X"], v["x"], v["width"], v["height"], 3, intr, max_iter=512)[0]["status"] == pro.RESECT_NO_MODEL
    for m in (0, 1, 3):
        assert pro.resect_view(v["X"][:m], v["x"][:m], v["width"], v["height"], 3, intr)[0]["status"] == pro.RESECT_TOO_FEW
    intr[0] = 0.0
    r, inl = pro.resect_view(v["X"], v["x"], v["width"], v["height"], 3, intr)
    assert r["status"] == pro.RESECT_NO_INTRINSIC and len(inl) == 0 and r["lm_termination"] == -1
    g = make_view(4, 300, outliers=0.2)
    intr = pro.intr8(g["focal"], g["ppx"], g["ppy"], g["disto"])
    a, ia = pro.resect_view(g["X"], g["x"], g["width"], g["height"], 3, intr, refine=False)
    b, ib = pro.resect_view(g["X"], g["x"], g["width"], g["height"], 3, intr)
    assert a["lm_termination"] == -1 and np.array_equal(a["rotation"], a["rotation_ransac"]) and np.array_equal(ia, ib)
    assert np.array_equal(a["rotation_ransac"], b["rotation_ransac"]) and not np.array_equal(a["rotation"], b["rotation"])
    c, ic = pro.resect_view(g["X"], g["x"], g["width"], g["height"], 3, intr, precision_px=1.0)
    assert c["status"] == pro.RESECT_OK and c["found_residual_precision"] <= 1.0


def _cost(v, pose, huber_a=16.0):
    r = project(v["model"], v["focal"], v["ppx"], v["ppy"], v["disto"], rodrigues(pose[:3]), pose[3:], v["X"]) - v["x"]
    s = (r * r).sum(1)
    return 0.5 * np.where(s > huber_a**2, 2 * huber_a * np.sqrt(s) - huber_a**2, s).sum()


def _start(v, rng):
    aa = np.zeros(3)
    # angle-axis of the true rotation through the oracle's residual-free route: perturb the truth directly
    from scipy.spatial.transform import Rotation
    aa = Rotation.from_matrix(v["R"]).as_rotvec()
    return np.concatenate([aa + rng.normal(size=3) * 2e-3, v["t"] + rng.normal(size=3) * 1e-2])


@pytest.mark.parametrize("model", [1, 2, 3, 4, 5])
def test_refinement_jacobian_and_optimum(model):
    from scipy.optimize import minimize
    rng = np.random.default_rng(model)
    v = make_view(60 + model, 300, model=model, noise=0.5)
    v["x"][:10] += 40.0  # residuals beyond the Huber width
    intr = pro.intr8(v["focal"], v["ppx"], v["ppy"], v["disto"])
    p0 = _start(v, rng)
    # the pose Jacobian the refinement uses against central differences of the numpy camera model
    _, J = po.ba_jacobian_model(model, intr[:6], intr[6:], p0, v["X"][17], v["x"][17])
    fd = np.zeros((2, 6))
    for k in range(6):
        d = np.zeros(6)
        d[k] = 1e-6
        f = [project(model, v["focal"], v["ppx"], v["ppy"], v["disto"], rodrigues((p0 + s * d)[:3]), (p0 + s * d)[3:], v["X"][17:18])[0]
             for s in (1, -1)]
        fd[:, k] = (f[0] - f[1]) / 2e-6
    assert np.abs(J[:, 6:12] - fd).max() <= 1e-5 * np.abs(fd).max()
    pose, s = pro.refine(model, intr, v["X"], v["x"], p0, function_tolerance=1e-14, parameter_tolerance=1e-14)
    assert s["termination"] in (1, 2, 3) and s["successful_steps"] >= 2
    assert abs(s["initial_cost"] - _cost(v, p0)) <= 1e-9 * s["initial_cost"]
    assert abs(s["final_cost"] - _cost(v, pose)) <= 1e-9 * s["final_cost"]
    best = minimize(lambda p: _cost(v, p), pose, method="Nelder-Mead", options=dict(xatol=1e-12, fatol=1e-14, maxiter=4000))
    assert s["final_cost"] - best.fun <= 1e-8 * s["final_cost"]


def test_refinement_reaches_the_truth_without_noise():
    rng = np.random.default_rng(9)
    for model in (1, 3, 4, 5):
        v = make_view(80 + model, 200, model=model, noise=0.0)
        intr = pro.intr8(v["focal"], v["ppx"], v["ppy"], v["disto"])
        pose, s = pro.refine(model, intr, v["X"], v["x"], _start(v, rng), function_tolerance=1e-30, parameter_tolerance=1e-16,
                             gradient_tolerance=1e-30, max_iterations=50)
        assert np.abs(rodrigues(pose[:3]) - v["R"]).max() <= 1e-9
        assert np.abs(pose[3:] - v["t"]).max() <= 1e-9 * max(1.0, np.abs(v["t"]).max())
        assert s["final_cost"] <= 1e-15
