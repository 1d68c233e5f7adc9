"""CPU oracle of the relative-pose step (oracle_relpose.cpp) against independent code: numpy's SVD, the synthetic
scene's true poses, cv2.recoverPose and scipy's least squares."""
import numpy as np
import pytest

from oracle import pyoracle_relpose as rpo
from regard3d_b200 import synth
from relpose_scenes import relative_truth, ring_truth, rotation_error_deg, two_view


def _numpy_motions(E):
    U, _, Vt = np.linalg.svd(E)
    if np.linalg.det(U) < 0:
        U[:, 2] *= -1
    if np.linalg.det(Vt) < 0:
        Vt[2] *= -1
    W = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1.0]])
    return [U @ W @ Vt, U @ W @ Vt, U @ W.T @ Vt, U @ W.T @ Vt], [U[:, 2], -U[:, 2], U[:, 2], -U[:, 2]]


def test_motions_from_essential_match_numpy_svd(oracle):
    rng = np.random.default_rng(0)
    for _ in range(300):
        R = synth._rodrigues(rng.normal(size=3))
        t = rng.normal(size=3)
        t /= np.linalg.norm(t)
        tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
        E = tx @ R * rng.uniform(0.1, 10.0)
        Rs, ts = rpo.motions_from_essential(E)
        Rn, tn = _numpy_motions(E)
        for k in range(4):   # as sets: the sign conventions of the two SVDs differ
            assert any(np.allclose(Rs[k], Rn[j], atol=1e-9) and np.allclose(ts[k], tn[j], atol=1e-9) for j in range(4))
        assert any(np.allclose(Rs[k], R, atol=1e-9) for k in range(4))
        for k in range(4):
            assert np.allclose(Rs[k] @ Rs[k].T, np.eye(3), atol=1e-12) and abs(np.linalg.det(Rs[k]) - 1) < 1e-12


def _Ks(sc):
    return np.array([[1.1 * max(int(w), int(h)), w / 2.0, h / 2.0] for w, h in zip(sc["widths"], sc["heights"])])


def test_ring_scene_recovers_the_true_relative_poses(oracle):
    sc = synth.make_scene(5, 1500, 64, "msurf", seed=41)
    Rs, ts = ring_truth(5, 1500, 64, "msurf", 41)
    pairs = synth.exhaustive_pairs(5)
    ofs, m = oracle.match_pairs(sc["descs"], sc["xys"], pairs, 0.8)
    for refine in (False, True):
        out, io, im = rpo.relative_poses(sc["xys"], sc["widths"], sc["heights"], _Ks(sc), pairs, ofs, m, refine=refine)
        assert (out["status"] == rpo.RELPOSE_OK).sum() >= 6
        for k, r in enumerate(out):
            if r["status"] != rpo.RELPOSE_OK:
                continue
            R, t = relative_truth(Rs, ts, int(r["I"]), int(r["J"]))
            tr = r["translation"] / np.linalg.norm(r["translation"])
            # a wrong motion is tens of degrees off; a narrow field of view couples small rotations with the baseline
            assert rotation_error_deg(R, r["rotation"]) < 2.0, (r["I"], r["J"])
            assert np.degrees(np.arccos(np.clip(tr @ t, -1, 1))) < 1.0
            assert io[k + 1] - io[k] == r["n_inliers"]
            if refine:
                assert r["ba_final_cost"] <= r["ba_initial_cost"] and r["ba_termination"] in (0, 1, 2, 3)
            else:
                assert r["ba_termination"] == -1 and abs(np.linalg.norm(r["translation"]) - 1) < 1e-12


def test_chosen_motion_agrees_with_cv2_recover_pose(oracle):
    cv2 = pytest.importorskip("cv2")
    xI, xJ, R, t, K = two_view(400, seed=3)
    r, inl = rpo.relative_pose(xI, xJ, 1920, 1080, 1920, 1080, np.r_[K, K], refine=False)
    assert r["status"] == rpo.RELPOSE_OK and len(inl) > 300
    Km = np.array([[K[0], 0, K[1]], [0, K[0], K[2]], [0, 0, 1.0]])
    E = r["E"]
    # the solver's E lives on bearing vectors: unit-norm rays, so it also constrains the normalised coordinates
    _, Rc, tc, _ = cv2.recoverPose(E, xI[inl].astype(np.float64), xJ[inl].astype(np.float64), Km)
    assert rotation_error_deg(Rc, r["rotation"]) < 1e-6
    assert np.allclose(tc.ravel() / np.linalg.norm(tc), r["translation"], atol=1e-6)
    assert rotation_error_deg(R, r["rotation"]) < 0.1


def test_refinement_matches_scipy_least_squares_with_huber(oracle):
    scipy_opt = pytest.importorskip("scipy.optimize")
    xI, xJ, R, t, K = two_view(60, seed=5)
    xJ[:3] += np.float32(30.0)   # three observations in the linear part of the Huber loss (|r| > 16 px)
    r0, inl = rpo.relative_pose(xI, xJ, 1920, 1080, 1920, 1080, np.r_[K, K], refine=False)
    r1, _ = rpo.relative_pose(xI, xJ, 1920, 1080, 1920, 1080, np.r_[K, K], refine=True)
    assert r0["status"] == rpo.RELPOSE_OK and r1["ba_termination"] in (1, 2, 3)
    a = 16.0

    def project(pose, X):
        Rm = synth._rodrigues(pose[:3])
        p = X @ Rm.T + pose[3:]
        return np.c_[K[0] * p[:, 0] / p[:, 2] + K[1], K[0] * p[:, 1] / p[:, 2] + K[2]]

    def residuals(v):
        # each 2-vector residual scaled by sqrt(rho(s) / s), s = |r|^2, Ceres' HuberLoss(a): 1/2 sum = Ceres' cost.
        # Camera I stays at (I, 0): the cost is gauge invariant, and the fixed gauge keeps scipy's Jacobian regular.
        poses, X = np.r_[np.zeros(6), v[:6]].reshape(2, 6), v[6:].reshape(-1, 3)
        out = []
        for c, x in ((0, xI), (1, xJ)):
            r = project(poses[c], X) - x
            s = (r ** 2).sum(1)
            w = np.where(s <= a * a, 1.0, np.sqrt((2 * a * np.sqrt(s) - a * a) / np.maximum(s, 1e-300)))
            out.append((r * w[:, None]).ravel())
        return np.concatenate(out)

    # the oracle's starting point: the unrefined motion and the DLT points
    c = np.clip((np.trace(r0["rotation"]) - 1) / 2, -1, 1)
    th = np.arccos(c)
    Rr = r0["rotation"]
    aa = th / (2 * np.sin(th)) * np.array([Rr[2, 1] - Rr[1, 2], Rr[0, 2] - Rr[2, 0], Rr[1, 0] - Rr[0, 1]])
    Kinv = np.linalg.inv(np.array([[K[0], 0, K[1]], [0, K[0], K[2]], [0, 0, 1.0]]))
    X0 = []
    for k in range(len(xI)):
        P1 = np.c_[np.eye(3), np.zeros(3)]
        P2 = np.c_[Rr, r0["translation"]]
        b1 = Kinv @ np.r_[xI[k], 1.0]
        b2 = Kinv @ np.r_[xJ[k], 1.0]
        A = np.stack([b1[0] * P1[2] - P1[0], b1[1] * P1[2] - P1[1], b2[0] * P2[2] - P2[0], b2[1] * P2[2] - P2[1]])
        X0.append(np.linalg.lstsq(A[:, :3], -A[:, 3], rcond=None)[0])
    v0 = np.r_[aa, r0["translation"], np.ravel(X0)]
    sol = scipy_opt.least_squares(residuals, v0, method="trf", x_scale="jac", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=5000)
    cost_scipy = 0.5 * (sol.fun ** 2).sum()
    assert abs(r1["ba_initial_cost"] - 0.5 * (residuals(v0) ** 2).sum()) < 1e-6 * r1["ba_initial_cost"]
    assert abs(r1["ba_final_cost"] - cost_scipy) < 1e-6 * cost_scipy
    # the same relative motion
    poses = np.r_[np.zeros(6), sol.x[:6]].reshape(2, 6)
    RI, RJ = synth._rodrigues(poses[0, :3]), synth._rodrigues(poses[1, :3])
    Rrel = RJ @ RI.T
    trel = poses[1, 3:] - Rrel @ poses[0, 3:]
    assert rotation_error_deg(Rrel, r1["rotation"]) < 1e-3
    assert np.allclose(trel / np.linalg.norm(trel), r1["translation"] / np.linalg.norm(r1["translation"]), atol=1e-4)


def test_rejection_statuses(oracle):
    xI, xJ, R, t, K = two_view(60, seed=7)
    Kp = np.r_[K, K]
    r, _ = rpo.relative_pose(xI[:5], xJ[:5], 1920, 1080, 1920, 1080, Kp)
    assert r["status"] == rpo.RELPOSE_TOO_FEW
    r, _ = rpo.relative_pose(xI, xJ, 1920, 1080, 1920, 1080, np.r_[K, 0.0, K[1:]])
    assert r["status"] == rpo.RELPOSE_NO_INTRINSIC
    rng = np.random.default_rng(1)
    r, _ = rpo.relative_pose(xI, xJ[rng.permutation(60)], 1920, 1080, 1920, 1080, Kp)
    assert r["status"] == rpo.RELPOSE_NO_MODEL
    # a consistent pair of only 12 matches: at most 12 inliers < 2.5 * 5
    r, _ = rpo.relative_pose(xI[:12], xJ[:12], 1920, 1080, 1920, 1080, Kp)
    assert r["status"] == rpo.RELPOSE_NO_MODEL
    r, inl = rpo.relative_pose(xI, xJ, 1920, 1080, 1920, 1080, Kp)
    assert r["status"] == rpo.RELPOSE_OK and r["n_inliers"] == len(inl) >= 13
    assert r["found_residual_precision"] <= 2.5
