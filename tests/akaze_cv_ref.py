"""CPU restatement of OpenCV 4's cv::AKAZE::detect (Regard3D's "AKAZE" detector) after the scale space.

The scale space is the Fast-AKAZE restatement's (oracle/pyoracle_akaze.py): Ldet, Lx and Ly of every level agree with
cv2's own (responses within a few ulp).  This module replays what cv::AKAZE does with them, each rule pinned against
cv2 4.13 by tests/test_oracle_akaze_cv.py (DESIGN.md 2.3):
  - candidates: 3x3 strict maxima above the threshold inside the level's border (the Fast-AKAZE candidates);
  - same-level pass over a per-level mask, candidates in raster order: the first kept point, in row-major order, of
    the window [y - r, y + r) x [x - r, x + r) with dx^2 + dy^2 <= r^2 (r = sigma_size) is cleared when the candidate
    is stronger, and the candidate dropped otherwise; without such a point the candidate is kept;
  - lower-level passes, i ascending: each kept point of level i looks at (x, y) * diff_ratio in level i - 1 within
    sigma_size_i * diff_ratio and clears the point found there when that one is weaker;
  - upper-level passes, i descending: each kept point of level i looks at (x, y) / diff_ratio (truncated) in level
    i + 1 within sigma_size_(i+1) and clears the weaker point found there.  Both passes scan their window forwards;
  - refinement: the 2x2 solve of Fast-AKAZE on every kept point in raster order, then x = (x + dx) ratio +
    0.5 (ratio - 1), size = 2 esigma derivative_factor, response = Ldet;
  - orientation: Fast-AKAZE's counting-sort window search (the oracle's orientation_sums), sampled at the placed
    point, and angle = hal::fastAtan2(maxY, maxX) in degrees.
Every float operation is float32 in the device's order, so libr3dgpu's R3D_DETECTOR_AKAZE agrees bit for bit.
"""
import numpy as np

from oracle import pyoracle_akaze as pa

f32 = np.float32
_DBL_EPS = f32(np.finfo(np.float64).eps)
# (i, j) of the 109 orientation samples, in the oracle's order
_SAMPLES = [(i, j) for i in range(-6, 7) for j in range(-6, 7) if i * i + j * j < 36]


def fast_atan2_deg(y, x):
    """hal::fastAtan2 (OpenCV 4.x fastAtan32f) in degrees, float32, elementwise."""
    y = np.asarray(y, f32)
    x = np.asarray(x, f32)
    r2d = f32(180 / np.pi)
    p1, p3 = f32(0.9997878412794807) * r2d, f32(-0.3258083974640975) * r2d
    p5, p7 = f32(0.1555786518463281) * r2d, f32(-0.04432655554792128) * r2d
    ax, ay = np.abs(x), np.abs(y)
    wide = ax >= ay
    with np.errstate(invalid="ignore", divide="ignore"):
        c = np.where(wide, ay / (ax + _DBL_EPS), ax / (ay + _DBL_EPS)).astype(f32)
    c2 = c * c
    poly = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c
    a = np.where(wide, poly, f32(90) - poly).astype(f32)
    a = np.where(x < 0, f32(180) - a, a).astype(f32)
    a = np.where(y < 0, f32(360) - a, a).astype(f32)
    return a


def candidates(ldet, border, threshold):
    """(y, x) of the 3x3 strict maxima above threshold inside border, raster order."""
    h, w = ldet.shape
    m = np.zeros((h, w), bool)
    if h - 2 * border <= 0 or w - 2 * border <= 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    c = ldet[1:-1, 1:-1]
    ok = c > f32(threshold)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dx or dy:
                ok &= c > ldet[1 + dy:h - 1 + dy, 1 + dx:w - 1 + dx]
    m[1:-1, 1:-1] = ok
    m[:border], m[h - border:], m[:, :border], m[:, w - border:] = False, False, False, False
    return np.nonzero(m)


_DISKS = {}


def _disk(r):
    if r not in _DISKS:
        d = np.arange(-r, r)
        _DISKS[r] = (d[:, None] ** 2 + d[None, :] ** 2) <= r * r
    return _DISKS[r]


def find_neighbor(mask, x, y, r):
    """find_neighbor_point: the first set pixel, row-major, of [y - r, y + r) x [x - r, x + r) within radius r."""
    hits = mask[y - r:y + r, x - r:x + r] & _disk(r)
    k = int(np.argmax(hits))
    if not hits.flat[k]:
        return None
    return y - r + k // (2 * r), x - r + k % (2 * r)


def extrema(levels, threshold):
    """The three passes over the per-level masks: returns (same, lower, upper), each a list of bool masks."""
    nl = len(levels)
    same = []
    for d in levels:
        L = d["Ldet"]
        r = int(d["level"]["sigma_size"])
        m = np.zeros(L.shape, bool)
        for y, x in zip(*candidates(L, int(d["level"]["border"]), threshold)):
            hit = find_neighbor(m, x, y, r)
            if hit is None:
                m[y, x] = True
            elif L[y, x] > L[hit]:
                m[hit] = False
                m[y, x] = True
        same.append(m)
    lower = [m.copy() for m in same]
    for i in range(1, nl):
        dr = int(levels[i]["level"]["ratio"] / levels[i - 1]["level"]["ratio"])
        r = int(levels[i]["level"]["sigma_size"]) * dr
        Li, Lp = levels[i]["Ldet"], levels[i - 1]["Ldet"]
        for y, x in zip(*np.nonzero(same[i])):
            hit = find_neighbor(lower[i - 1], x * dr, y * dr, r)
            if hit is not None and Li[y, x] > Lp[hit]:
                lower[i - 1][hit] = False
    upper = [m.copy() for m in lower]
    for i in range(nl - 2, -1, -1):
        dr = int(levels[i + 1]["level"]["ratio"] / levels[i]["level"]["ratio"])
        r = int(levels[i + 1]["level"]["sigma_size"])
        Li, Ln = levels[i]["Ldet"], levels[i + 1]["Ldet"]
        for y, x in zip(*np.nonzero(lower[i])):
            hit = find_neighbor(upper[i + 1], x // dr, y // dr, r)
            if hit is not None and Li[y, x] > Ln[hit]:
                upper[i + 1][hit] = False
    return same, lower, upper


def refine(ldet, level, index, ys, xs):
    """Subpixel refinement of kept points (raster order) of one level: keypoint_dtype, rejected points left out."""
    l = ldet
    c, e, w_, n, s = l[ys, xs], l[ys, xs + 1], l[ys, xs - 1], l[ys - 1, xs], l[ys + 1, xs]
    Dx = f32(0.5) * (e - w_)
    Dy = f32(0.5) * (s - n)
    Dxx = e + w_ - f32(2) * c
    Dyy = s + n - f32(2) * c
    Dxy = f32(0.25) * (l[ys + 1, xs + 1] + l[ys - 1, xs - 1] - l[ys - 1, xs + 1] - l[ys + 1, xs - 1])
    b0, b1 = -Dx, -Dy
    d = Dxx.astype(np.float64) * Dyy - Dxy.astype(np.float64) * Dxy
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        dx = np.where(d != 0, ((b0.astype(np.float64) * Dyy - b1.astype(np.float64) * Dxy) * inv).astype(f32), f32(0))
        dy = np.where(d != 0, ((b1.astype(np.float64) * Dxx - b0.astype(np.float64) * Dxy) * inv).astype(f32), f32(0))
    dx, dy = dx.astype(f32), dy.astype(f32)
    ok = (np.abs(dx) <= 1) & (np.abs(dy) <= 1)
    ratio = f32(level["ratio"])
    out = np.zeros(int(ok.sum()), pa.keypoint_dtype)
    off = f32(0.5) * (ratio - f32(1))
    out["x"] = (xs[ok].astype(f32) + dx[ok]) * ratio + off
    out["y"] = (ys[ok].astype(f32) + dy[ok]) * ratio + off
    out["size"] = f32(level["esigma"]) * f32(1.5) * f32(2)
    out["response"] = c[ok]
    out["octave"] = int(level["octave"])
    out["class_id"] = index
    return out


def orientation_sums(kps, levels):
    """The oracle's orientation_sums (Fast-AKAZE's Compute_Main_Orientation up to the angle) for many keypoints at
    once: (n, 2) float32 (maxX, maxY)."""
    n = len(kps)
    out = np.zeros((n, 2), f32)
    g = pa.gauss25()
    wgt = np.array([g[abs(i), abs(j)] for i, j in _SAMPLES], f32)
    si = np.array([i for i, _ in _SAMPLES])
    sj = np.array([j for _, j in _SAMPLES])
    quantum = f32(2.0 * np.pi / 42)
    for li, d in enumerate(levels):
        sel = np.nonzero(kps["class_id"] == li)[0]
        if not len(sel):
            continue
        k = kps[sel]
        ratio = f32(d["level"]["ratio"])
        scale = (f32(0.5) * k["size"] / ratio + f32(0.5)).astype(np.int64)
        x0 = (k["x"] / ratio + f32(0.5)).astype(np.int64)
        y0 = (k["y"] / ratio + f32(0.5)).astype(np.int64)
        py = y0[:, None] + si[None, :] * scale[:, None]
        px = x0[:, None] + sj[None, :] * scale[:, None]
        rx = (wgt[None, :] * d["Lx"][py, px]).astype(f32)
        ry = (wgt[None, :] * d["Ly"][py, px]).astype(f32)
        key = (pa.fast_atan2(ry, rx) / quantum).astype(np.int64)
        best_n = np.full(len(sel), -np.inf, np.float32)
        bx = np.zeros(len(sel), f32)
        by = np.zeros(len(sel), f32)
        idx = np.arange(109)
        for sn in range(42):
            # window sn: slices sn .. sn + 6 (mod 42), summed slice by slice, each slice in descending sample order
            rank = (key - sn) % 42
            inside = (rank < 7) & (key < 42)
            order = np.argsort(np.where(inside, rank * 128 + (108 - idx)[None, :], 1 << 20), axis=1, kind="stable")
            sx = np.zeros(len(sel), f32)
            sy = np.zeros(len(sel), f32)
            ins = np.take_along_axis(inside, order, 1)
            ox = np.take_along_axis(rx, order, 1)
            oy = np.take_along_axis(ry, order, 1)
            for p in range(109):
                if not ins[:, p].any():
                    break
                sx = np.where(ins[:, p], sx + ox[:, p], sx).astype(f32)
                sy = np.where(ins[:, p], sy + oy[:, p], sy).astype(f32)
            nrm = (sx * sx + sy * sy).astype(f32)
            better = nrm > best_n if sn else np.ones(len(sel), bool)
            best_n = np.where(better, nrm, best_n).astype(f32)
            bx = np.where(better, sx, bx).astype(f32)
            by = np.where(better, sy, by).astype(f32)
        out[sel, 0] = bx
        out[sel, 1] = by
    return out


def detect(img, threshold=7e-4, octaves=4, sublevels=4, levels=False):
    """cv::AKAZE::detect on one float32 gray image in [0, 1]: keypoint_dtype in cv2's order (levels ascending, raster
    order within a level).  levels=True also returns the oracle's per-level dicts with the three masks added
    ("same", "lower", "upper")."""
    _, lv, _ = pa.detect(img, threshold, octaves, sublevels, levels=True)
    same, lower, upper = extrema(lv, threshold)
    parts = []
    for i, d in enumerate(lv):
        ys, xs = np.nonzero(upper[i])
        parts.append(refine(d["Ldet"], d["level"], i, ys, xs))
        d.update(same=same[i], lower=lower[i], upper=upper[i])
    kps = np.concatenate(parts) if parts else np.zeros(0, pa.keypoint_dtype)
    ori = orientation_sums(kps, lv)
    kps["angle"] = fast_atan2_deg(ori[:, 1], ori[:, 0])
    return (kps, lv) if levels else kps


# named exceptions to the cv2 bars (tests/test_oracle_akaze_cv.py explains them), by (w, h, seed, threshold)
POSITION_EXCEPTIONS = {(640, 480, 21, 1e-4): 1.5e-3, (641, 479, 5, 1e-4): 1.5e-3}
RESPONSE_EXCEPTIONS = {(641, 479, 5, 1e-4): 1.5e-5}
ANGLE_EXCEPTIONS = {(640, 480, 23, 1e-4): 1}


def assert_matches_cv2(got, exp, case):
    assert len(got) == len(exp), (case, len(got), len(exp))
    assert np.array_equal(got["class_id"], exp["class_id"]), case
    assert np.array_equal(got["octave"], exp["octave"]), case
    assert np.array_equal(got["size"], exp["size"]), case
    rel = np.abs(got["response"].astype(np.float64) - exp["response"]) / np.abs(exp["response"].astype(np.float64))
    assert rel.max(initial=0) <= RESPONSE_EXCEPTIONS.get(case, 1e-5), (case, rel.max())
    dpos = np.maximum(np.abs(got["x"].astype(np.float64) - exp["x"]), np.abs(got["y"].astype(np.float64) - exp["y"]))
    assert dpos.max(initial=0) <= POSITION_EXCEPTIONS.get(case, 1e-3), (case, dpos.max())
    da = np.abs((got["angle"].astype(np.float64) - exp["angle"] + 180.0) % 360.0 - 180.0)
    assert int((da > 0.01).sum()) <= ANGLE_EXCEPTIONS.get(case, 0), (case, np.sort(da)[-3:])
