"""Synthetic relative translations with known camera centres and rotations for the translation-averaging tests and
bench."""
import numpy as np

from regard3d_b200 import capi
from rotavg_scenes import axis_angle, banded_ring, complete_edges, random_rotation  # noqa: F401


def make_problem(n, edges, noise_deg=0.0, outlier_frac=0.0, seed=0, scale_range=(0.5, 2.0), extent=10.0):
    """Ground-truth centres Cs (uniform in a cube of side 2 * extent, so not collinear) and rotations Rs; one relative
    pose record per edge (I, J) with R_IJ = R_J R_I^T and t_IJ = R_J (C_I - C_J) times a random factor in scale_range,
    its direction turned by |N(0, noise_deg)| degrees about a random axis; half of the records are stored reversed
    (J, I); outlier edges get a uniformly random direction.  Returns (records, Rs, Cs, outlier mask)."""
    rng = np.random.default_rng(seed)
    Rs = np.array([random_rotation(rng) for _ in range(n)])
    Cs = rng.uniform(-extent, extent, size=(n, 3))
    I, J, R, T, out = [], [], [], [], []
    for (i, j) in edges:
        if rng.random() < 0.5:
            i, j = j, i
        t = Rs[j] @ (Cs[i] - Cs[j]) * rng.uniform(*scale_range)
        if noise_deg > 0:
            t = axis_angle(rng.standard_normal(3), abs(rng.normal(0.0, noise_deg))) @ t
        bad = rng.random() < outlier_frac
        if bad:
            d = rng.standard_normal(3)
            t = d / np.linalg.norm(d) * np.linalg.norm(t)
        out.append(bad)
        I.append(i); J.append(j); R.append(Rs[j] @ Rs[i].T); T.append(t)
    rel = capi.relative_pose_records(I, J, np.array(R).reshape(-1, 3, 3))
    rel["translation"] = np.array(T).reshape(-1, 3)
    return rel, Rs, Cs, np.array(out, bool)


def similarity_align(C_est, C_true):
    """Umeyama: the similarity (s, R, t) minimising |s R C_est + t - C_true|; returns the aligned C_est."""
    mu_e, mu_t = C_est.mean(0), C_true.mean(0)
    E, T = C_est - mu_e, C_true - mu_t
    U, S, Vt = np.linalg.svd(T.T @ E)
    D = np.eye(3)
    if np.linalg.det(U @ Vt) < 0:
        D[2, 2] = -1
    Rm = U @ D @ Vt
    s = np.trace(np.diag(S) @ D) / (E ** 2).sum()
    return s * E @ Rm.T + mu_t


def aligned_error(C_est, C_true, kept):
    """Largest distance between the kept estimated centres (after a similarity alignment) and the truth, over the
    diameter of the true kept centres."""
    ids = np.nonzero(kept)[0]
    A = similarity_align(C_est[ids], C_true[ids])
    diam = max(np.linalg.norm(C_true[ids] - C_true[ids].mean(0), axis=1).max() * 2, 1e-300)
    return float(np.linalg.norm(A - C_true[ids], axis=1).max() / diam)
