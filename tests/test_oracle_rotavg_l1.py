"""The CPU restatement of r3d_rotation_averaging_l1 (rotavg_l1_ref.py) against independent references: its primal-dual
l1 solver against HiGHS, exact recovery without noise, robustness to gross outliers against the L2 method, and its
IRLS fixed point against a step recomputed from scratch."""
import numpy as np
import pytest
import scipy.optimize
from scipy.spatial.transform import Rotation

import rotavg_l1_ref as ref
from oracle import pyoracle_rotavg as rpo
from rotavg_scenes import axis_angle, complete_edges, gauge_error_fro, make_problem

# Robustness scene: a 40-view complete graph, 0.5 degree noise, 20 % gross outliers (20..180 degrees), all kept by a
# 180 degree triplet threshold (every cycle but an exact half turn is valid).  Measured with the restatement on seeds
# 41..43 at 15 % and 20 % outliers (threshold 181 degrees): L1 0.23 .. 0.37 degrees from the truth, L2 15.6 .. 22.6.
ROBUST_L1_BOUND_DEG = 0.5
ROBUST_L2_OVER_L1 = 20.0


def robust_scene(seed=42):
    n = 40
    rel, Rs, _ = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.2, seed=seed)
    return rel, Rs, n


def _deg(R, Rs, kept):
    return np.degrees(gauge_error_fro(R, Rs, kept) / np.sqrt(2))


def _dense_A(ab, m):
    A = np.zeros((3 * len(ab), 3 * m))
    for e, (a, b) in enumerate(ab):
        for k in range(3):
            A[3 * e + k, 3 * a + k] = -1.0
            A[3 * e + k, 3 * b + k] = 1.0
    return A[:, 3:]  # the held view's columns dropped


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_pd_solver_reaches_the_highs_optimum(seed):
    """min |A x - b|_1 on a random graph (a ring plus chords; small residuals and 20 % gross ones): the primal-dual
    solution's objective is above HiGHS' optimum by at most the final surrogate duality gap, which is below pdtol."""
    rng = np.random.default_rng(seed)
    m = 12
    E = sorted({(i, (i + 1) % m) if i < (i + 1) % m else ((i + 1) % m, i) for i in range(m)}
               | {tuple(sorted(rng.choice(m, 2, replace=False))) for _ in range(20)})
    ab = np.array(E, np.int64)
    b = rng.normal(0.0, 0.02, (len(ab), 3))
    bad = rng.random(len(ab)) < 0.2
    b[bad] = rng.uniform(-1.0, 1.0, (bad.sum(), 3))
    x, st = ref.l1_regression(ab, b, m)
    A = _dense_A(ab, m)
    nv, nr = A.shape[1], A.shape[0]
    I = np.eye(nr)
    lp = scipy.optimize.linprog(np.r_[np.zeros(nv), np.ones(nr)], A_ub=np.block([[A, -I], [-A, -I]]),
                                b_ub=np.r_[b.ravel(), -b.ravel()], bounds=[(None, None)] * nv + [(0, None)] * nr,
                                method="highs")
    assert lp.status == 0
    got = np.abs(A @ x[1:].ravel() - b.ravel()).sum()
    assert 0.0 < st["sdg"] < ref.PD_TOL and not st["stuck"]
    assert lp.fun - 1e-9 <= got <= lp.fun + st["sdg"], (got, lp.fun, st["sdg"])


def test_noise_free_recovery():
    """Without noise the truth comes back to 1e-10 after the gauge, from the spanning tree and from a start 10 degrees
    off every view (a wrong sign in the update R <- R exp([x]x) or in A would not converge)."""
    n = 20
    rel, Rs, _ = make_problem(n, complete_edges(n), seed=5)
    r, vk, _, _, S = ref.rotation_averaging_l1(rel, n, tolerance=1e-12, irls_max_iterations=50)
    assert S["termination"] == 0 and gauge_error_fro(r, Rs, vk) < 1e-10
    _, _, _, _, ab, Rab, views = ref.kept_problem(rel, n)
    rng = np.random.default_rng(6)
    truth = np.array([Rs[v] @ Rs[views[0]].T for v in views])
    start = np.array([truth[0]] + [Rv @ axis_angle(rng.standard_normal(3), 10.0) for Rv in truth[1:]])
    R, S = ref.solve(ab, Rab, len(views), tolerance=1e-12, irls_max_iterations=50, start=start)
    assert S["termination"] == 0 and S["l1_iterations"] >= 2
    assert max(np.linalg.norm(R[v] - truth[v]) for v in range(len(views))) < 1e-10


def test_robust_to_gross_outliers():
    """Every outlier survives the triplet test (threshold 180 degrees): L1 stays within ROBUST_L1_BOUND_DEG of
    the truth and beats the L2 method (orc_rotation_averaging, refined) by ROBUST_L2_OVER_L1."""
    rel, Rs, n = robust_scene()
    r1, v1, e1, _, S1 = ref.rotation_averaging_l1(rel, n, max_angular_error_deg=180.0)
    r2, v2, e2, _, _ = rpo.rotation_averaging(rel, n, max_angular_error_deg=180.0)
    assert e1.all() and np.array_equal(v1, v2) and S1["termination"] == 0
    d1, d2 = _deg(r1, Rs, v1), _deg(r2, Rs, v2)
    assert d1 < ROBUST_L1_BOUND_DEG and d2 > ROBUST_L2_OVER_L1 * d1, (d1, d2)


def test_irls_fixed_point():
    """One IRLS step from the returned rotations, recomputed from scratch (scipy's rotation log, the dense A, W and
    normal equations), moves no view by more than the tolerance."""
    n = 60
    rel, _, _ = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.15, seed=21)
    r, vk, ek, _, S = ref.rotation_averaging_l1(rel, n)
    assert S["termination"] == 0 and S["irls_iterations"] >= 1
    views = np.nonzero(vk)[0]
    local = {int(v): i for i, v in enumerate(views)}
    ab, bres = [], []
    for k in np.nonzero(ek)[0]:
        I, J, Rij = int(rel["I"][k]), int(rel["J"][k]), rel["rotation"][k].reshape(3, 3)
        ab.append((local[I], local[J]))
        bres.append(Rotation.from_matrix(r[J].T @ Rij @ r[I]).as_rotvec())  # row +1 at J, -1 at I
    ab, bres = np.array(ab), np.array(bres).ravel()
    A = np.zeros((len(bres), 3 * len(views)))
    for e, (i, j) in enumerate(ab):
        for c in range(3):
            A[3 * e + c, 3 * i + c] -= 1.0
            A[3 * e + c, 3 * j + c] += 1.0
    A = A[:, 3:]
    s2 = np.radians(5.0) ** 2
    w = s2 / (bres ** 2 + s2) ** 2
    x = np.linalg.solve(A.T @ (w[:, None] * A), A.T @ (w * bres))
    assert np.abs(x).max() <= ref.DEFAULTS["tolerance"]


def test_no_component_and_invalid_options():
    rel, _, _ = make_problem(6, [(i, i + 1) for i in range(5)], noise_deg=0.3, seed=3)
    r, vk, ek, sup, S = ref.rotation_averaging_l1(rel, 6)
    assert S["success"] == 0 and S["termination"] == -1 and not r.any() and not vk.any() and not ek.any()
    for bad in (dict(l1_max_iterations=0), dict(irls_max_iterations=-1), dict(tolerance=0.0), dict(tolerance=np.nan),
                dict(irls_sigma_deg=0.0)):
        with pytest.raises(ValueError):
            ref.rotation_averaging_l1(rel, 6, **bad)
