"""The CPU oracle of what follows the SfM engine (oracle/oracle_export.cpp) against independent restatements: the
ColorizeTracks plan against plain Python dicts and sets, the undistortion against a numpy float64 evaluation of every
camera model, the coloured PLY against a Python writer.  No GPU."""
import math

import numpy as np
import pytest

from export_scenes import python_plan, random_scene

pe = pytest.importorskip("oracle.pyoracle_export")


@pytest.fixture(scope="module", autouse=True)
def _built():
    pe.build()


def _plan(views, landmarks):
    return pe.colorize_plan(*pe.flatten(views, landmarks))


@pytest.mark.parametrize("seed,kw", [
    (1, dict()),
    (2, dict(n_views=40, n_lm=60, max_obs=2)),         # many views, few tracks: equal counts in most rounds
    (3, dict(n_views=6, n_lm=500, max_obs=1)),         # one-observation tracks only
    (4, dict(n_views=25, n_lm=2000, max_obs=6, posed_frac=0.4)),
    (5, dict(n_views=3, n_lm=40, max_obs=3, edge_frac=0.9, sizes=((1, 1), (2, 3)))),
])
def test_plan_equals_python_restatement(seed, kw):
    views, landmarks = random_scene(seed, **kw)
    got = _plan(views, landmarks)
    exp = python_plan(views, landmarks)
    for g, e in zip(got, exp):
        assert np.array_equal(g, e)
    unposed = {v["id_view"] for v in views if not v["has_pose"]}
    assert unposed and not unposed & set(got[0].tolist())
    # every landmark takes its pixel from an observation in the view of its round
    for l, r, (x, y) in zip(sorted(landmarks, key=lambda a: a["id"]), got[1], got[2]):
        ob = [o for o in l["obs"] if o[0] == got[0][r]]
        assert len(ob) == 1 and (int(ob[0][2]), int(ob[0][3])) == (x, y)


def test_plan_tie_takes_first_view_in_id_order():
    views = [dict(id_view=v, width=8, height=8, has_pose=True) for v in (7, 3, 11)]
    landmarks = [dict(id=0, X=[0, 0, 0], obs=[(3, 0, 1.0, 1.0), (11, 0, 2.0, 2.0)]),
                 dict(id=1, X=[0, 0, 0], obs=[(7, 0, 3.0, 3.0), (11, 1, 4.0, 4.0)]),
                 dict(id=2, X=[0, 0, 0], obs=[(3, 1, 5.0, 5.0), (7, 1, 6.0, 6.0)])]
    rv, lr, lp = _plan(views, landmarks)
    assert rv.tolist() == [3, 7] and lr.tolist() == [0, 1, 0] and lp.tolist() == [[1, 1], [3, 3], [5, 5]]


@pytest.mark.parametrize("bad", ["empty_track", "x_minus_one", "x_width", "y_height", "nan"])
def test_plan_rejects_undefined_inputs(bad):
    views = [dict(id_view=0, width=10, height=6, has_pose=True)]
    obs = {"empty_track": [], "x_minus_one": [(0, 0, -1.0, 2.0)], "x_width": [(0, 0, 10.0, 2.0)],
           "y_height": [(0, 0, 2.0, 6.0)], "nan": [(0, 0, float("nan"), 2.0)]}[bad]
    landmarks = [dict(id=0, X=[0, 0, 0], obs=[(0, 0, 9.999, 5.999)]), dict(id=1, X=[0, 0, 0], obs=obs)]
    with pytest.raises(pe.OracleError):
        _plan(views, landmarks)


# ---- undistortion -------------------------------------------------------------------------------------------------
def _numpy_undistort(model, f, ppx, ppy, disto, rgb):
    """UndistortImage with every step in numpy float64 (np.arctan, np.hypot), the sampler as DESIGN.md 2.4 reads it.
    Returns the image and, per pixel, whether the result may legitimately differ from another correct evaluation by
    one: a sample coordinate within 1e-9 of an integer or an image edge, or of a float32 rounding tie, or a channel
    value before the conversion within 1e-6 of an integer."""
    h, w = rgb.shape[:2]
    k = np.zeros(5)
    k[:len(disto)] = disto
    if model == 1:
        return rgb.copy(), np.zeros((h, w), bool)
    j, i = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    x, y = (i - ppx) / f, (j - ppy) / f
    if model == 5:
        r = np.hypot(x, y)
        th = np.arctan(r)
        t2 = th * th
        t3 = t2 * th
        t4 = t2 * t2
        t5 = t4 * th
        t7 = t3 * t3 * th
        t8 = t4 * t4
        t9 = t8 * th
        thd = th + k[0] * t3 + k[1] * t5 + k[2] * t7 + k[3] * t9
        with np.errstate(divide="ignore", invalid="ignore"):
            cd = np.where(r > 1e-8, thd * (1.0 / r), 1.0)
        xd, yd = x * cd, y * cd
    else:
        r2 = x * x + y * y
        r4 = r2 * r2
        r6 = r4 * r2
        if model == 4:
            kd = k[0] * r2 + k[1] * r4 + k[2] * r6
            xd = x + (x * kd + (k[4] * (r2 + 2 * x * x) + 2 * k[3] * x * y))
            yd = y + (y * kd + (k[3] * (r2 + 2 * y * y) + 2 * k[4] * x * y))
        else:
            rc = 1.0 + k[0] * r2 + k[1] * r4 + k[2] * r6 if model == 3 else 1.0 + k[0] * r2
            xd, yd = x * rc, y * rc
    dx, dy = f * xd + ppx, f * yd + ppy
    inside = (dx > -1) & (dx < w) & (dy > -1) & (dy < h)
    fx, fy = dx.astype(np.float32), dy.astype(np.float32)
    flx, fly = np.floor(fx), np.floor(fy)
    ax, ay = fx - flx, fy - fly
    cx, cy = (np.float32(1) - ax, ax), (np.float32(1) - ay, ay)
    gx, gy = flx.astype(np.int64), fly.astype(np.int64)
    acc = np.zeros((h, w, 3))
    tw = np.zeros((h, w))
    for a in (0, 1):
        for b in (0, 1):
            yy, xx = gy + a, gx + b
            ok = inside & (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
            wt = (cx[b] * cy[a]).astype(np.float64)
            pix = rgb[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)].astype(np.float64)
            acc = acc + np.where(ok[..., None], pix * wt[..., None], 0.0)
            tw = tw + np.where(ok, wt, 0.0)
    keep = inside & (tw > 0.2)
    with np.errstate(divide="ignore", invalid="ignore"):
        val = np.where((tw != 1.0)[..., None], acc / tw[..., None], acc)
    out = np.where(keep[..., None], np.clip(np.nan_to_num(val), 0, 255).astype(np.uint8), 0).astype(np.uint8)

    def near_int(v):
        return np.abs(v - np.round(v)) < 1e-9

    def near_f32_tie(v):  # the float32 cast could round the other way
        lo = v.astype(np.float32).astype(np.float64)
        nxt = np.nextafter(v.astype(np.float32), np.where(v >= lo, np.inf, -np.inf).astype(np.float32)).astype(np.float64)
        return np.abs(v - 0.5 * (lo + nxt)) < 1e-9 * np.maximum(1.0, np.abs(v))

    edge = (np.abs(dx + 1) < 1e-9) | (np.abs(dx - w) < 1e-9) | (np.abs(dy + 1) < 1e-9) | (np.abs(dy - h) < 1e-9)
    amb = near_int(dx) | near_int(dy) | edge | near_f32_tie(dx) | near_f32_tie(dy)
    amb |= keep & (np.abs(val - np.round(val)) < 1e-6).any(-1)
    amb |= np.abs(tw - 0.2) < 1e-9
    return out, amb


MODELS = {
    "pinhole": (1, ()),
    "radial1": (2, (-0.21,)),
    "radial3": (3, (-0.25, 0.12, -0.03)),
    "brown": (4, (-0.18, 0.05, -0.01, 0.002, -0.003)),
    "fisheye": (5, (0.05, -0.02, 0.01, -0.004)),
    "radial3_zero": (3, (0.0, 0.0, 0.0)),
    "radial1_strong": (2, (0.9,)),               # maps most of the frame outside: black borders
    "fisheye_strong": (5, (0.6, 0.3, 0.1, 0.05)),
}


@pytest.mark.parametrize("name", sorted(MODELS))
@pytest.mark.parametrize("size", [(1, 1), (3, 2), (97, 61), (641, 479)])
def test_undistort_equals_numpy_reference(name, size):
    model, disto = MODELS[name]
    w, h = size
    rng = np.random.default_rng(w * 7 + h + model)
    rgb = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
    f, ppx, ppy = 0.9 * max(w, h) + 0.3, w / 2.0 - 0.37, h / 2.0 + 0.21
    got = pe.undistort_image(model, f, ppx, ppy, disto, rgb)
    exp, amb = _numpy_undistort(model, f, ppx, ppy, disto, rgb)
    diff = np.abs(got.astype(int) - exp.astype(int)).max(-1)
    n_amb = int((diff > 0).sum())
    assert diff.max() <= 1 and not ((diff > 0) & ~amb).any(), \
        "%d pixels differ, %d of them outside the documented ambiguities" % (n_amb, int(((diff > 0) & ~amb).sum()))
    print("%s %dx%d: %d of %d pixels differ by one at a documented ambiguity" % (name, w, h, n_amb, w * h))
    if model == 1:
        assert np.array_equal(got, rgb)
    if name.endswith("strong") and w > 10:
        assert (got.reshape(-1, 3) == 0).all(-1).any(), "expected black borders"


def test_undistort_rejects_unknown_model():
    with pytest.raises(pe.OracleError):
        pe.undistort_image(6, 10.0, 1.0, 1.0, (), np.zeros((2, 2, 3), np.uint8))


# ---- FinalColorized.ply -------------------------------------------------------------------------------------------
def python_ply(X, colors, centers):
    lines = ["ply", "format ascii 1.0", "element vertex %d" % (len(X) + len(centers)), "property double x", "property double y",
             "property double z", "property uchar red", "property uchar green", "property uchar blue", "end_header"]
    out = "\n".join(lines) + "\n"
    for k, p in enumerate(X):
        c = "255 255 255" if colors is None else "%d %d %d" % tuple(int(v) for v in colors[k])
        out += "%.16f %.16f %.16f %s\n" % (p[0], p[1], p[2], c)
    for p in centers:
        out += "%.16f %.16f %.16f 0 255 0\n" % (p[0], p[1], p[2])
    return out.encode()


def _ply_case(seed):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(50, 3)) * 10.0 ** rng.integers(-8, 8, size=(50, 1))
    X[0] = (0.0, -0.0, 1e300)
    X[1] = (-1e-300, 123456789.123456789, -7.5)
    colors = rng.integers(0, 256, size=(50, 3), dtype=np.uint8)
    centers = rng.normal(size=(4, 3))
    return X, colors, centers


@pytest.mark.parametrize("with_colors", [True, False])
def test_ply_bytes_equal_python_writer(tmp_path, with_colors):
    X, colors, centers = _ply_case(8)
    colors = colors if with_colors else None
    path = str(tmp_path / "FinalColorized.ply")
    pe.write_colorized_ply(path, X, colors, centers)
    assert open(path, "rb").read() == python_ply(X, colors, centers)


def test_library_ply_writer_equals_oracle(tmp_path, r3dlib):
    """r3d_sfm_write_colorized_ply is host code: the same bytes as the oracle's std::ofstream writer."""
    X, colors, centers = _ply_case(9)
    sd = r3dlib.SfmData()
    sd.add_view(0, "a.jpg", 10, 10)
    sd.add_intrinsic(0, 3, 10, 10, 12.0, 5.0, 5.0)
    ids = np.random.default_rng(2).choice(10000, len(X), replace=False)
    order = np.argsort(ids)
    for k in range(len(X)):
        sd.add_landmark(int(ids[k]), X[k].tolist(), [(0, k, 1.0, 1.0)])
    for p, c in enumerate(centers):
        sd.add_pose(10 * (len(centers) - p), np.eye(3), c)  # pose ids in reverse: written in id order
    cen = centers[::-1]
    for cols in (colors[order], None):
        a, b = str(tmp_path / "lib.ply"), str(tmp_path / "orc.ply")
        sd.write_colorized_ply(a, cols)
        pe.write_colorized_ply(b, X[order], cols, cen)
        assert open(a, "rb").read() == open(b, "rb").read()
    with pytest.raises(r3dlib.R3DError) as e:
        sd.write_colorized_ply(str(tmp_path / "missing" / "x.ply"))
    assert e.value.code == -4 and "missing" in str(e.value)
    assert math.isfinite(X[1][1])
