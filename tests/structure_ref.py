"""An independent float64 / long-double reference of the structure steps (sfm_structure.cu and its CPU oracle), numpy only:
undistortion of every camera model, triangulation from known poses, and the two outlier filters the engines run after
bundle adjustment.  The camera model is `resection_scenes.distort`; nothing here calls library or oracle code.

Observations are flat arrays in landmark order: landmark l owns observations ofs[l] .. ofs[l + 1].  A camera is
(model, disto, f, ppx, ppy, R, t) with R, t world -> camera; per-observation arrays `cam` index a list of cameras."""
import numpy as np

from resection_scenes import distort

LD = np.longdouble


# ---- undistortion ---------------------------------------------------------------------------------------------------
def undistort_normalised(model, disto, xd, yd, tol=1e-12):
    """Inverse of `distort` on normalised coordinates by Newton with a central-difference Jacobian, until the forward
    residual is below 1e-12 (asserted, not assumed from an iteration count)."""
    xd = np.asarray(xd, np.float64)
    yd = np.asarray(yd, np.float64)
    if model == 1:
        return xd.copy(), yd.copy()
    xu, yu = xd.copy(), yd.copy()
    h = 1e-7
    for _ in range(60):
        fx, fy = distort(model, disto, xu, yu)
        gx, gy = fx - xd, fy - yd
        if max(np.abs(gx).max(initial=0.0), np.abs(gy).max(initial=0.0)) < 1e-15:
            break
        ax, ay = distort(model, disto, xu + h, yu)
        bx, by = distort(model, disto, xu - h, yu)
        cx, cy = distort(model, disto, xu, yu + h)
        dx, dy = distort(model, disto, xu, yu - h)
        j00, j10 = (ax - bx) / (2 * h), (ay - by) / (2 * h)
        j01, j11 = (cx - dx) / (2 * h), (cy - dy) / (2 * h)
        det = j00 * j11 - j01 * j10
        xu = xu - (j11 * gx - j01 * gy) / det
        yu = yu - (j00 * gy - j10 * gx) / det
    fx, fy = distort(model, disto, xu, yu)
    res = max(np.abs(fx - xd).max(initial=0.0), np.abs(fy - yd).max(initial=0.0))
    assert res < tol, "undistortion did not converge: forward residual %.3g" % res
    return xu, yu


def undistort_pixels(cams, cam, xy):
    """Undistorted pixels (n x 2, float64) of observations xy (n x 2) seen by cameras cams[cam]."""
    cam = np.asarray(cam)
    xy = np.asarray(xy, np.float64)
    out = np.empty_like(xy)
    for c in np.unique(cam):
        m = cam == c
        model, disto, f, ppx, ppy = cams[c][:5]
        xu, yu = undistort_normalised(model, disto, (xy[m, 0] - ppx) / f, (xy[m, 1] - ppy) / f)
        out[m, 0] = ppx + f * xu
        out[m, 1] = ppy + f * yu
    return out


# ---- triangulation ----------------------------------------------------------------------------------------------------
def _projection(cams, cam):
    """K [R | t] per observation, long double (n x 3 x 4)."""
    P = np.empty((len(cam), 3, 4), LD)
    for c in np.unique(cam):
        _, _, f, ppx, ppy, R, t = cams[c]
        K = np.array([[f, 0, ppx], [0, f, ppy], [0, 0, 1]], LD)
        P[cam == c] = K @ np.c_[np.asarray(R, LD), np.asarray(t, LD)]
    return P


def _segments(ofs):
    ofs = np.asarray(ofs, np.int64)
    n = np.diff(ofs)
    return ofs, n, np.repeat(np.arange(len(n)), n)


def _inv3(a):
    """Adjugate inverse of a batch of 3 x 3 matrices (long double)."""
    c = np.empty_like(a)
    for i in range(3):
        for j in range(3):
            r = [k for k in range(3) if k != j]
            s = [k for k in range(3) if k != i]
            c[:, i, j] = (-1) ** (i + j) * (a[:, r[0], s[0]] * a[:, r[1], s[1]] - a[:, r[0], s[1]] * a[:, r[1], s[0]])
    det = np.einsum("nj,nj->n", a[:, 0, :], c[:, :, 0])
    return c / det[:, None, None]


def triangulate(cams, ofs, cam, xy_ud):
    """`Triangulation::compute(3)`: iteratively re-weighted inhomogeneous DLT (weights 1 / depth of the previous pass),
    three passes; ok when the landmark has two observations and its smallest depth after the last pass is positive.
    Returns (X float64 n x 3, ok)."""
    ofs, n, owner = _segments(ofs)
    P = _projection(cams, np.asarray(cam))
    x = np.asarray(xy_ud, LD)
    L = len(n)
    X = np.zeros((L, 3), LD)
    w = np.ones(len(owner), LD)
    good = n >= 2
    zmin = np.zeros(L, LD)
    for it in range(3):
        v1 = w[:, None] * (P[:, 0, :3] - x[:, :1] * P[:, 2, :3])
        v2 = w[:, None] * (P[:, 1, :3] - x[:, 1:] * P[:, 2, :3])
        b1 = w * (x[:, 0] * P[:, 2, 3] - P[:, 0, 3])
        b2 = w * (x[:, 1] * P[:, 2, 3] - P[:, 1, 3])
        AtA = np.zeros((L, 3, 3), LD)
        Atb = np.zeros((L, 3), LD)
        np.add.at(AtA, owner, v1[:, :, None] * v1[:, None, :] + v2[:, :, None] * v2[:, None, :])
        np.add.at(Atb, owner, v1 * b1[:, None] + v2 * b2[:, None])
        AtA[~good] = np.eye(3, dtype=LD)
        X = np.einsum("nij,nj->ni", _inv3(AtA), Atb)
        z = np.einsum("nj,nj->n", P[:, 2, :3], X[owner]) + P[:, 2, 3]
        w = 1 / z
        zmin = np.full(L, np.inf, LD)
        np.minimum.at(zmin, owner, z)
    return X.astype(np.float64), good & (zmin > 0)


def sensitivity(cams, ofs, cam, X):
    """Per landmark, the smallest singular value of d(normalised projections) / dX over its observations: a change of
    the undistorted observations of norm d (normalised units) moves the least-squares point by about d / sigma."""
    ofs, n, owner = _segments(ofs)
    cam = np.asarray(cam)
    J = np.zeros((len(owner), 2, 3))
    for c in np.unique(cam):
        m = cam == c
        R, t = np.asarray(cams[c][5]), np.asarray(cams[c][6])
        p = X[owner[m]] @ R.T + t
        z = p[:, 2:]
        J[m, 0] = (R[0] - p[:, :1] / z * R[2]) / z
        J[m, 1] = (R[1] - p[:, 1:2] / z * R[2]) / z
    JtJ = np.zeros((len(n), 3, 3))
    np.add.at(JtJ, owner, np.einsum("nki,nkj->nij", J, J))
    JtJ[n < 2] = np.eye(3)
    return np.sqrt(np.maximum(np.linalg.eigvalsh(JtJ)[:, 0], 1e-300))


def bisection_error(model, disto, f, ppx, ppy, xy):
    """Bound (normalised units) on the error of upstream's radial K1 / K3 undistortion (bisection on r^2 that stops at a
    bracket of 1e-8; below r^2 = 2e-7 the first 5 % bracket is already that narrow and decides)."""
    if model not in (2, 3) or not any(disto[:3]):
        return np.zeros(len(xy))
    r2 = ((xy[:, 0] - ppx) / f) ** 2 + ((xy[:, 1] - ppy) / f) ** 2
    dr2 = np.where(r2 < 2e-7, 0.06 * r2, 1e-8)            # |error of r_u^2|, with margin on the 5 % bracket
    return np.where(r2 > 0, dr2 / (2 * np.sqrt(np.maximum(r2, 1e-300)) * 0.9), 0.0)  # -> error of r_u


def point_bound(ofs, obs_err, sigma):
    """Bound on |dX| from per-observation errors (normalised units, per coordinate): 2 |d|_2 / sigma."""
    ofs, n, owner = _segments(ofs)
    s = np.zeros(len(n))
    np.add.at(s, owner, 2.0 * np.asarray(obs_err) ** 2)
    return 2.0 * np.sqrt(s) / sigma


# ---- outlier filters ------------------------------------------------------------------------------------------------
def residuals(cams, ofs, cam, xy, X):
    """Pixel residual norm of every observation through the camera model, long double."""
    ofs, n, owner = _segments(ofs)
    cam = np.asarray(cam)
    xy = np.asarray(xy, LD)
    X = np.asarray(X, LD)
    out = np.zeros(len(cam), LD)
    for c in np.unique(cam):
        m = cam == c
        model, disto, f, ppx, ppy, R, t = cams[c]
        p = X[owner[m]] @ np.asarray(R, LD).T + np.asarray(t, LD)
        xd, yd = distort(model, [LD(d) for d in disto], p[:, 0] / p[:, 2], p[:, 1] / p[:, 2])
        out[m] = np.hypot(LD(ppx) + LD(f) * xd - xy[m, 0], LD(ppy) + LD(f) * yd - xy[m, 1])
    return out


def max_ray_angle(cams, cam_list, X):
    """Largest angle (degrees, long double) between two rays X - C of the cameras in cam_list; 0 for fewer than two."""
    X = np.asarray(X, LD)
    rays = []
    for c in cam_list:
        R, t = np.asarray(cams[c][5], LD), np.asarray(cams[c][6], LD)
        u = X + R.T @ t                                   # X - C, C = -R^T t
        rays.append(u / np.sqrt(np.sum(u * u)))
    best = LD(0)
    for a in range(len(rays)):
        for b in range(a + 1, len(rays)):
            cs = min(max(np.sum(rays[a] * rays[b]), LD(-1)), LD(1))
            best = max(best, np.degrees(np.arccos(cs)))
    return best


def remove_outliers(cams, ofs, cam, xy, X, thr, min_track_length, min_angle_deg, rel=1e-9):
    """RemoveOutliers_PixelResidualError(thr, min_track_length) then RemoveOutliers_AngleError(min_angle_deg) on what it
    left, as upstream runs them back to back.  Returns dict:
      keep        {landmark index: kept observation indices}
      rm_obs, rm_lm
      ambiguous   landmark indices whose outcome depends on a residual or angle within `rel` of its threshold
    """
    ofs = np.asarray(ofs, np.int64)
    res = residuals(cams, ofs, cam, xy, X)
    near = np.abs(res - LD(thr)) <= LD(rel) * LD(thr)
    keep, amb = {}, set()
    rm_obs = rm_lm = 0
    for l in range(len(ofs) - 1):
        obs = np.arange(ofs[l], ofs[l + 1])
        if near[obs].any():
            amb.add(l)
        kept = obs[res[obs] <= LD(thr)]
        rm_obs += len(obs) - len(kept)
        if len(kept) == 0 or len(kept) < min_track_length:
            rm_lm += 1
            continue
        ang = max_ray_angle(cams, [cam[o] for o in kept], X[l])
        if abs(ang - LD(min_angle_deg)) <= LD(rel) * LD(min_angle_deg):
            amb.add(l)
        if ang < LD(min_angle_deg):
            rm_lm += 1
            continue
        keep[l] = kept
    return dict(keep=keep, rm_obs=rm_obs, rm_lm=rm_lm, ambiguous=amb, residual=res)


# ---- scene helpers ----------------------------------------------------------------------------------------------------
def look_at(C, target=(0.0, 0.0, 0.0), up=(0.0, 1.0, 0.0)):
    """R (world -> camera, rows x y z) and t of a camera at C whose optical axis points at target."""
    C = np.asarray(C, np.float64)
    z = np.asarray(target, np.float64) - C
    z /= np.linalg.norm(z)
    x = np.cross(np.asarray(up, np.float64), z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    return R, -R @ C


def sphere_centres(rng, n, radius, spread=0.8):
    """n camera centres on a cap of a sphere around the origin (polar angle up to `spread` rad from -z)."""
    th = rng.uniform(0.0, spread, n)
    ph = rng.uniform(0.0, 2 * np.pi, n)
    return radius * np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), -np.cos(th)], 1)
