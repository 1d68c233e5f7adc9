"""Seeded resection scenes shared by the oracle and the GPU tests: points in front of a camera, pixel noise, an outlier
fraction, any of the five camera models."""
import numpy as np

# distortion coefficients of realistic size per camera model (openMVG EINTRINSIC 1..5)
DISTO = {1: (), 2: (-0.08,), 3: (-0.12, 0.05, -0.01), 4: (-0.1, 0.04, -0.008, 0.0015, -0.001), 5: (-0.03, 0.006, -0.001, 0.0002)}


def rodrigues(aa):
    aa = np.asarray(aa, float)
    th = np.linalg.norm(aa)
    if th < 1e-12:
        return np.eye(3)
    k = aa / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def distort(model, disto, xu, yu):
    """The forward camera model on normalised coordinates (openMVG's add_disto), written independently of the library."""
    d = list(disto) + [0.0] * 5
    r2 = xu * xu + yu * yu
    if model == 1:
        return xu, yu
    if model == 5:
        r = np.sqrt(r2)
        th = np.arctan(r)
        thd = th + d[0] * th**3 + d[1] * th**5 + d[2] * th**7 + d[3] * th**9
        c = np.where(r > 1e-8, thd / np.maximum(r, 1e-300), 1.0)
        return xu * c, yu * c
    k2, k3 = (d[1], d[2]) if model >= 3 else (0.0, 0.0)
    c = 1 + d[0] * r2 + k2 * r2**2 + k3 * r2**3
    xd, yd = xu * c, yu * c
    if model == 4:
        t1, t2 = d[3], d[4]
        xd = xd + t2 * (r2 + 2 * xu * xu) + 2 * t1 * xu * yu
        yd = yd + t1 * (r2 + 2 * yu * yu) + 2 * t2 * xu * yu
    return xd, yd


def project(model, focal, ppx, ppy, disto, R, t, X):
    p = X @ R.T + t
    xd, yd = distort(model, disto, p[:, 0] / p[:, 2], p[:, 1] / p[:, 2])
    return np.stack([ppx + focal * xd, ppy + focal * yd], 1)


def make_view(seed, M, model=3, outliers=0.0, noise=0.3, width=2000, height=1500, focal=None):
    """One view: dict with X (M x 3), x (M x 2 pixels), the true R, t, the inlier mask and the camera."""
    rng = np.random.default_rng(seed)
    focal = 1.1 * max(width, height) if focal is None else focal
    ppx, ppy = width / 2.0 + rng.uniform(-5, 5), height / 2.0 + rng.uniform(-5, 5)
    disto = DISTO[model]
    R = rodrigues(rng.normal(size=3) * 0.6)
    C = rng.normal(size=3) * 2.0
    t = -R @ C
    # points in the camera frame, spread over the image and over depth, then moved to the world
    u = rng.uniform(0.05 * width, 0.95 * width, M)
    v = rng.uniform(0.05 * height, 0.95 * height, M)
    z = rng.uniform(4.0, 12.0, M)
    pc = np.stack([(u - ppx) / focal * z, (v - ppy) / focal * z, z], 1)
    X = (pc - t) @ R
    x = project(model, focal, ppx, ppy, disto, R, t, X) + rng.normal(size=(M, 2)) * noise
    inlier = np.ones(M, bool)
    n_out = int(round(outliers * M))
    if n_out:
        bad = rng.choice(M, n_out, replace=False)
        x[bad] = np.stack([rng.uniform(0, width, n_out), rng.uniform(0, height, n_out)], 1)
        inlier[bad] = False
    return dict(X=X, x=x, R=R, t=t, C=C, inlier=inlier, model=model, width=width, height=height, focal=focal, ppx=ppx, ppy=ppy,
                disto=disto, scale=float(np.abs(X).max()) if M else 1.0)


def make_batch(seed, n_views, M, models=(3,), **kw):
    """n_views views; M: an int or one count per view."""
    Ms = [M] * n_views if np.isscalar(M) else list(M)
    return [make_view(seed * 1000 + v, Ms[v], model=models[v % len(models)], **kw) for v in range(n_views)]


def rotation_angle_deg(Ra, Rb):
    c = (np.trace(Ra.T @ Rb) - 1.0) / 2.0
    return float(np.degrees(np.arccos(np.clip(c, -1.0, 1.0))))
