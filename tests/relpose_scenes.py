"""Two-view scenes with a known relative pose for the relative-pose tests."""
import numpy as np

from regard3d_b200 import synth


def ring_truth(n_images, n_feats, dim, kind="msurf", seed=0):
    """The camera rotations / translations synth.make_scene draws for these arguments (its stored angle-axis poses
    are unreliable near 180 degrees, so the tests replay the generator instead)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    n_points = max(16, int(n_feats * 1.5))
    rng.uniform([0, 0, 0], [10, 10, 4], size=(n_points, 3))
    synth._descriptor_family(kind, dim, rng, n_points)
    _, Rs, ts = synth.ring_cameras(n_images, rng)
    return Rs, ts


def relative_truth(Rs, ts, I, J):
    R = Rs[J] @ Rs[I].T
    t = ts[J] - R @ ts[I]
    return R, t / np.linalg.norm(t)


def rotation_error_deg(Ra, Rb):
    c = np.clip((np.trace(Ra.T @ Rb) - 1.0) / 2.0, -1.0, 1.0)
    return float(np.degrees(np.arccos(c)))


def two_view(n, seed, baseline=(1.0, 0.1, 0.05), rot=(0.02, -0.15, 0.03), noise_px=0.5, outlier_frac=0.0, w=1920, h=1080,
             f=None):
    """n correspondences of random points seen by camera I = (I, 0) and camera J = (R(rot), baseline): positions (n, 2)
    float32 in both views, the true (R, t), K."""
    rng = np.random.default_rng(seed)
    f = 1.1 * max(w, h) if f is None else f
    R = synth._rodrigues(np.asarray(rot, float))
    t = np.asarray(baseline, float)
    X = np.c_[rng.uniform(-4, 4, 4 * n), rng.uniform(-2.5, 2.5, 4 * n), rng.uniform(6, 14, 4 * n)]
    xI, vI = synth.project(np.eye(3), np.zeros(3), X, f, w, h)
    xJ, vJ = synth.project(R, t, X, f, w, h)
    keep = np.nonzero(vI & vJ)[0][:n]
    assert len(keep) == n
    xI = xI[keep] + noise_px * rng.standard_normal((n, 2))
    xJ = xJ[keep] + noise_px * rng.standard_normal((n, 2))
    bad = rng.random(n) < outlier_frac
    xJ[bad] = np.c_[rng.uniform(0, w, bad.sum()), rng.uniform(0, h, bad.sum())]
    K = np.array([f, w / 2.0, h / 2.0])
    return xI.astype(np.float32), xJ.astype(np.float32), R, t, K
