"""The CPU oracle of the structure steps (oracle/oracle_sfm.cpp) against the independent float64 / long-double reference
in structure_ref.py, on every camera model: triangulation from known poses and the per-landmark outlier checks."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import structure_ref as sr
from resection_scenes import DISTO, project

FOCAL, PPX, PPY = 2200.0, 1000.5, 749.75


def _ext(model, disto):
    """intrinsics_ext of one group: t1 t2 (Brown), k4 0 (fisheye), zeros otherwise."""
    d = list(disto) + [0.0] * 5
    return [d[3], d[4]] if model in (4, 5) else [0.0, 0.0]


def _scene(model, seed, n_cams=4, M=2000):
    """n_cams cameras around the origin with one intrinsic of `model`, M points seen by all of them (noise-free)."""
    rng = np.random.default_rng(seed)
    cams = []
    for C in sr.sphere_centres(rng, n_cams, 8.0):
        R, t = sr.look_at(C, rng.normal(size=3) * 0.2)
        cams.append((model, DISTO[model], FOCAL, PPX, PPY, R, t))
    X = rng.uniform(-2.0, 2.0, (M, 3))
    ofs = np.arange(M + 1, dtype=np.uint64) * n_cams
    cam = np.tile(np.arange(n_cams), M)
    xy = np.concatenate([project(model, FOCAL, PPX, PPY, DISTO[model], cams[c][5], cams[c][6], X[l:l + 1])
                         for l in range(M) for c in range(n_cams)])
    return cams, X, ofs, cam, xy


def _oracle_args(cams, model):
    poses = np.array([np.r_[Rotation.from_matrix(c[5]).as_rotvec(), c[6]] for c in cams])
    intr = np.array([[FOCAL, PPX, PPY] + (list(DISTO[model]) + [0.0] * 3)[:3]])
    return poses, np.zeros(len(cams), np.uint32), intr, np.array([model], np.uint8), np.array([_ext(model, DISTO[model])])


def _point_tolerance(cams, model, ofs, cam, xy, X):
    """1e-9 relative, plus what the K1 / K3 bisection may move the point by."""
    sigma = sr.sensitivity(cams, ofs, cam, X)
    e = sr.bisection_error(model, DISTO[model], FOCAL, PPX, PPY, xy)
    return 1e-9 * np.linalg.norm(X, axis=1) + sr.point_bound(ofs, e, sigma)


@pytest.mark.parametrize("model", [1, 2, 3, 4, 5])
def test_triangulation_matches_the_reference(oracle, model):
    cams, Xt, ofs, cam, xy = _scene(model, 300 + model)
    Xr, okr = sr.triangulate(cams, ofs, cam, sr.undistort_pixels(cams, cam, xy))
    assert okr.all()
    # the reference itself: noise-free float64 pixels land on the truth
    assert (np.linalg.norm(Xr - Xt, axis=1) <= 1e-9 * np.linalg.norm(Xt, axis=1)).all()
    poses, cam_intr, intr, im, ext = _oracle_args(cams, model)
    Xo, oko = oracle.triangulate_landmarks(ofs, cam, xy, poses, cam_intr, intr, intr_model=im, intr_ext=ext)
    assert oko.all()
    err = np.linalg.norm(Xo - Xr, axis=1)
    tol = _point_tolerance(cams, model, ofs, cam, xy, Xr)
    assert (err <= tol).all(), "model %d: max rel. error %.3g" % (model, (err / np.linalg.norm(Xr, axis=1)).max())
    if model in (1, 4, 5):
        assert (tol <= 1.01e-9 * np.linalg.norm(Xr, axis=1)).all()


@pytest.mark.parametrize("model", [1, 2, 3, 4, 5])
def test_landmark_checks_match_the_reference(oracle, model):
    cams, Xt, ofs, cam, xy = _scene(model, 400 + model, M=1500)
    rng = np.random.default_rng(500 + model)
    thr = 4.0
    # half of the observations moved to a residual within 0.01 .. 3 px of the threshold, on either side
    off = np.where(rng.uniform(size=len(xy)) < 0.5, 0.0, thr + rng.choice([-1, 1], len(xy)) * rng.uniform(0.01, 3.0, len(xy)))
    ang = rng.uniform(0, 2 * np.pi, len(xy))
    xy = xy + off[:, None] * np.stack([np.cos(ang), np.sin(ang)], 1)
    ref = sr.remove_outliers(cams, ofs, cam, xy, Xt, thr, 2, 0.0)
    poses, cam_intr, intr, im, ext = _oracle_args(cams, model)
    keep, max_angle = oracle.landmark_checks(ofs, cam, xy, poses, cam_intr, intr, Xt, thr, intr_model=im, intr_ext=ext)
    near = np.abs(ref["residual"] - thr) <= 1e-9 * thr
    assert near.sum() <= 2
    assert np.array_equal(keep[~near], (ref["residual"] <= thr)[~near])
    assert 0 < (~keep).sum() < len(keep)
    for l in range(len(ofs) - 1):
        a = sr.max_ray_angle(cams, cam[int(ofs[l]):int(ofs[l + 1])], Xt[l])
        assert abs(max_angle[l] - float(a)) <= 1e-9 * max(1.0, float(a)), l
