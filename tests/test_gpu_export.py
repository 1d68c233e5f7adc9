"""-m gpu: the colour plan (r3d_sfm_colorize_plan) and the undistortion (r3d_undistort_images) against the CPU oracle
(oracle/oracle_export.cpp), bit for bit; SfmData.colorize + write_colorized_ply against the oracle's file."""
import ctypes as C

import numpy as np
import pytest

from export_scenes import ba_scene, image_for, oracle_plan, random_scene, to_sfm

pytestmark = pytest.mark.gpu
pe = pytest.importorskip("oracle.pyoracle_export")


def _check_plan(ctx, r3dlib, views, landmarks):
    sd = to_sfm(r3dlib, views, landmarks)
    got = ctx.colorize_plan(sd)
    exp = oracle_plan(views, landmarks)
    for name, g, e in zip(("round_view", "lm_round", "lm_pixel"), got, exp):
        assert np.array_equal(g, e), name
    return got


@pytest.mark.parametrize("seed,kw", [
    (11, dict()),
    (12, dict(n_views=40, n_lm=60, max_obs=2)),
    (13, dict(n_views=6, n_lm=500, max_obs=1)),
    (14, dict(n_views=25, n_lm=3000, max_obs=6, posed_frac=0.4)),
    (15, dict(n_views=3, n_lm=40, max_obs=3, edge_frac=0.9, sizes=((1, 1), (2, 3)))),
])
def test_plan_small_scenes(gpu_ctx, r3dlib, seed, kw):
    _check_plan(gpu_ctx, r3dlib, *random_scene(seed, **kw))


def test_plan_many_views_global_counts(gpu_ctx, r3dlib):
    """More views than the per-CTA shared-memory histogram holds: the counts go to global memory directly."""
    _check_plan(gpu_ctx, r3dlib, *random_scene(16, n_views=12500, n_lm=5000, max_obs=3, sizes=((32, 24),)))


def test_plan_million_observations_with_forced_ties(gpu_ctx, r3dlib):
    views, landmarks = ba_scene(n_cams=100, n_pts=100000, obs_per_pt=5, seed=29, twins=True)
    assert sum(len(l["obs"]) for l in landmarks) >= 900000
    rv, _, _ = _check_plan(gpu_ctx, r3dlib, views, landmarks)
    assert (rv < 100).all(), "a twin of higher id never wins its tie"


def test_plan_rejections(gpu_ctx, r3dlib):
    views = [dict(id_view=0, width=10, height=6, has_pose=True), dict(id_view=1, width=10, height=6, has_pose=False)]
    good = dict(id=0, X=[0, 0, 0], obs=[(0, 0, 9.999, 5.999)])
    for bad in ([], [(0, 0, -1.0, 2.0)], [(0, 0, 10.0, 2.0)], [(0, 0, 2.0, 6.0)], [(0, 0, float("nan"), 1.0)],
                [(1, 0, 1.0, 1.0)]):  # the last: a view without a pose
        sd = to_sfm(r3dlib, views, [good, dict(id=1, X=[0, 0, 0], obs=bad)])
        with pytest.raises(r3dlib.R3DError) as e:
            gpu_ctx.colorize_plan(sd)
        assert e.value.code == -1
    empty = to_sfm(r3dlib, views, [])
    rv, lr, lp = gpu_ctx.colorize_plan(empty)
    assert len(rv) == 0 and len(lr) == 0 and lp.shape == (0, 2)


def test_colorize_and_ply_equal_oracle(gpu_ctx, r3dlib, tmp_path):
    views, landmarks = random_scene(21, n_views=10, n_lm=800, max_obs=4)
    sd = to_sfm(r3dlib, views, landmarks)
    size = {v["id_view"]: (v["width"], v["height"]) for v in views}
    reads = []

    def read_rgb(v):
        reads.append(v)
        return image_for(v, *size[v])

    colors = sd.colorize(gpu_ctx, read_rgb)
    rv, lr, lp = oracle_plan(views, landmarks)
    assert reads == rv.tolist()
    exp_colors = np.zeros((len(lr), 3), np.uint8)
    for k in range(len(lr)):
        v = int(rv[lr[k]])
        exp_colors[k] = image_for(v, *size[v])[lp[k, 1], lp[k, 0]]
    assert np.array_equal(colors, exp_colors)
    a, b = str(tmp_path / "FinalColorized.ply"), str(tmp_path / "oracle.ply")
    sd.write_colorized_ply(a, colors)
    lms = sorted(landmarks, key=lambda l: l["id"])
    cen = [p["center"] for p in sd.poses()]
    pe.write_colorized_ply(b, np.array([l["X"] for l in lms]), exp_colors, np.array(cen))
    assert open(a, "rb").read() == open(b, "rb").read()


# ---- undistortion -------------------------------------------------------------------------------------------------
MODELS = {
    "pinhole": (1, ()),
    "radial1": (2, (-0.21,)),
    "radial3": (3, (-0.25, 0.12, -0.03)),
    "brown": (4, (-0.18, 0.05, -0.01, 0.002, -0.003)),
    "fisheye": (5, (0.05, -0.02, 0.01, -0.004)),
    "radial3_zero": (3, (0.0, 0.0, 0.0)),
    "radial1_strong": (2, (0.9,)),
    "brown_strong": (4, (0.8, 0.4, 0.2, 0.05, -0.04)),
    "fisheye_strong": (5, (0.6, 0.3, 0.1, 0.05)),
}


def _intr(name, w, h):
    model, disto = MODELS[name]
    return dict(model=model, focal=0.9 * max(w, h) + 0.3, ppx=w / 2.0 - 0.37, ppy=h / 2.0 + 0.21, disto=disto)


def _img(w, h, seed):
    return np.random.default_rng(seed).integers(0, 256, size=(h, w, 3), dtype=np.uint8)


def _oracle(d, img):
    return pe.undistort_image(d["model"], d["focal"], d["ppx"], d["ppy"], d["disto"], img)


@pytest.mark.parametrize("size", [(1, 1), (3, 2), (641, 479), (4000, 3000)])
def test_undistort_equals_oracle(gpu_ctx, size):
    w, h = size
    names = sorted(MODELS)
    img = _img(w, h, w + h)
    intr = [_intr(n, w, h) for n in names]
    got = gpu_ctx.undistort_images(intr, [img] * len(names))
    t = gpu_ctx.last_undistort_timing
    assert t["images"] == len(names) and t["copied"] == 1 and t["kernel_launches"] == len(names) - 1
    for n, d, g in zip(names, intr, got):
        assert np.array_equal(g, _oracle(d, img)), n
        if n == "pinhole":
            assert np.array_equal(g, img)
        if n.endswith("strong") and w > 100:
            assert (g.reshape(-1, 3) == 0).all(-1).mean() > 0.01, "expected black borders"


def test_undistort_mixed_batch(gpu_ctx):
    sizes = [(641, 479), (1, 1), (3, 2), (1920, 1080), (97, 61), (640, 480), (33, 1)]
    names = sorted(MODELS)
    rng = np.random.default_rng(5)
    imgs, intr = [], []
    for k in range(14):
        w, h = sizes[k % len(sizes)]
        imgs.append(_img(w, h, 100 + k))
        intr.append(_intr(names[int(rng.integers(len(names)))], w, h))
    got = gpu_ctx.undistort_images(intr, imgs)
    for k, (d, img, g) in enumerate(zip(intr, imgs, got)):
        assert np.array_equal(g, _oracle(d, img)), k
    again = gpu_ctx.undistort_images(intr, imgs)
    assert all(np.array_equal(a, b) for a, b in zip(got, again))


def test_undistort_rejects_invalid_arguments(gpu_ctx, r3dlib):
    lib, h = r3dlib.lib(), gpu_ctx._h
    img = np.zeros((4, 5, 3), np.uint8)
    out = np.zeros_like(img)
    intr = (r3dlib.SfmIntrinsic * 1)(r3dlib.SfmIntrinsic(0, 3, 5, 4, 5.0, 2.5, 2.0, (C.c_double * 5)()))
    src = (C.c_void_p * 1)(img.ctypes.data)
    dst = (C.c_void_p * 1)(out.ctypes.data)
    ws, hs = np.array([5], np.uint32), np.array([4], np.uint32)
    zero = np.array([0], np.uint32)
    p = r3dlib._p
    assert lib.r3d_undistort_images(h, 1, intr, src, p(ws), p(hs), dst, None) == 0
    assert lib.r3d_undistort_images(h, 0, None, None, None, None, None, None) == 0
    assert lib.r3d_undistort_images(None, 1, intr, src, p(ws), p(hs), dst, None) == -1
    for args in ((None, src, p(ws), p(hs), dst), (intr, None, p(ws), p(hs), dst), (intr, src, None, p(hs), dst),
                 (intr, src, p(ws), None, dst), (intr, src, p(ws), p(hs), None),
                 (intr, (C.c_void_p * 1)(None), p(ws), p(hs), dst), (intr, src, p(ws), p(hs), (C.c_void_p * 1)(None)),
                 (intr, src, p(zero), p(hs), dst), (intr, src, p(ws), p(zero), dst)):
        assert lib.r3d_undistort_images(h, 1, *args, None) == -1
    for model in (0, 6, -3):
        intr[0].model = model
        assert lib.r3d_undistort_images(h, 1, intr, src, p(ws), p(hs), dst, None) == -1
    with pytest.raises(ValueError):
        gpu_ctx.undistort_images([_intr("radial3", 5, 4)], [np.zeros((4, 5), np.uint8)])
