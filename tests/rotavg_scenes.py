"""Synthetic relative rotations with known global rotations for the rotation-averaging tests and bench."""
import itertools

import numpy as np

from regard3d_b200 import capi


def random_rotation(rng):
    q = rng.standard_normal(4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def axis_angle(axis, deg):
    a = np.asarray(axis, float)
    a = a / np.linalg.norm(a)
    t = np.radians(deg)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(t) * K + (1 - np.cos(t)) * K @ K


def angle_deg(R):
    return float(np.degrees(np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1))))


def complete_edges(n):
    return list(itertools.combinations(range(n), 2))


def banded_ring(n, k):
    return sorted({(min(i, (i + d) % n), max(i, (i + d) % n)) for i in range(n) for d in range(1, k + 1)})


def make_problem(n, edges, noise_deg=0.0, outlier_frac=0.0, seed=0, outlier_min_deg=20.0):
    """Ground truth Rs (non-commuting, uniform), one relative pose record per edge (I, J) with R_IJ = R_J R_I^T times a
    noise rotation, half of them stored reversed (J, I) with R^T; outlier edges replaced by a rotation at least
    outlier_min_deg off.  Returns (records, Rs, outlier mask)."""
    rng = np.random.default_rng(seed)
    Rs = np.array([random_rotation(rng) for _ in range(n)])
    I, J, R, out = [], [], [], []
    for (i, j) in edges:
        Rij = Rs[j] @ Rs[i].T
        if noise_deg > 0:
            Rij = axis_angle(rng.standard_normal(3), abs(rng.normal(0.0, noise_deg))) @ Rij
        bad = rng.random() < outlier_frac
        if bad:
            Rij = axis_angle(rng.standard_normal(3), rng.uniform(outlier_min_deg, 180.0)) @ Rij
        out.append(bad)
        if rng.random() < 0.5:
            I.append(i); J.append(j); R.append(Rij)
        else:
            I.append(j); J.append(i); R.append(Rij.T)
    return capi.relative_pose_records(I, J, np.array(R)), Rs, np.array(out, bool)


def gauge_error_deg(R_est, R_true, kept):
    """Largest angle between R_est[i] and R_true[i] R_true[r]^T over the kept views, r = the lowest kept view."""
    ids = np.nonzero(kept)[0]
    r = ids[0]
    return max(angle_deg(R_est[i].T @ (R_true[i] @ R_true[r].T)) for i in ids)


def gauge_error_fro(R_est, R_true, kept):
    """Largest Frobenius distance between R_est[i] and R_true[i] R_true[r]^T over the kept views (r = lowest kept view);
    ~ sqrt(2) x the angle in radians, without arccos' loss of precision near zero."""
    ids = np.nonzero(kept)[0]
    r = ids[0]
    return max(float(np.linalg.norm(R_est[i] - R_true[i] @ R_true[r].T)) for i in ids)
