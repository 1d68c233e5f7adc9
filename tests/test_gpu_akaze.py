"""Fast-AKAZE on the device against the CPU restatement (oracle/oracle_akaze.cpp): every level's Lt, Lsmooth, Lx, Ly,
Ldet and kcontrast, the candidate lists and deletion flags of the three extrema passes, and every keypoint field in
upstream order, bit for bit."""
import numpy as np
import pytest

from akaze_scenes import scene
from oracle import pyoracle_akaze as pa

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from regard3d_b200 import capi
    c = capi.Context((0,))
    yield c
    c.close()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _same_keypoints(got, exp):
    assert len(got) == len(exp)
    assert got.tobytes() == exp.tobytes(), "keypoints differ from the oracle's"


def _compare_levels(ctx, img, threshold, stats=None):
    exp_k, exp_l, _ = pa.detect(img, threshold, levels=True, stats=stats)
    got_l = ctx.debug_akaze_levels(img, threshold=threshold)
    assert len(got_l) == len(exp_l)
    for i, (g, e) in enumerate(zip(got_l, exp_l)):
        assert g["level"].tobytes() == e["level"].tobytes(), "level %d record" % i
        assert np.float32(g["kcontrast"]) == np.float32(e["kcontrast"]), "level %d kcontrast" % i
        for name in pa.ARRAYS:
            assert np.array_equal(_bits(g[name]), _bits(e[name])), "level %d %s differs" % (i, name)
        assert g["candidates"].tobytes() == e["candidates"].tobytes(), "level %d same-level pass" % i
        assert np.array_equal(g["deleted_lower"], e["deleted_lower"]), "level %d lower-level pass" % i
        assert np.array_equal(g["deleted_upper"], e["deleted_upper"]), "level %d upper-level pass" % i
    got_k = ctx.akaze_detect([img], threshold=threshold)[0]
    _same_keypoints(got_k, exp_k)
    return exp_k, exp_l


@pytest.mark.parametrize("w,h,threshold", [
    (640, 480, 1e-3),
    (641, 479, 1e-3),     # odd sides: OpenCV's fractional-area halving at every octave
    (150, 120, 1e-4),     # one octave: the next would be narrower than 80 px
    (100, 100, 1e-4),     # the level list ends mid-octave on the border rule
    (640, 480, 1e-4),
    (640, 480, 1e-2),
])
def test_levels_and_keypoints_bit_identical(ctx, w, h, threshold):
    stats = {}
    k, lv = _compare_levels(ctx, scene(w, h, seed=w + h), threshold, stats)
    if (w, h, threshold) == (640, 480, 1e-3):
        # the scene exercises in-place replacement in the same-level pass, both deletion passes and the |d| > 1
        # rejection
        assert stats["replaced"] > 0 and stats["rejected"] > 0
        assert any(l["deleted_lower"].any() for l in lv)
        assert any((l["deleted_upper"] & ~l["deleted_lower"]).any() for l in lv)
        assert len(k) < sum(int((~l["deleted_upper"]).sum()) for l in lv)


def test_large_image(ctx):
    img = scene(4000, 3000, seed=7)
    _compare_levels(ctx, img, 1e-3)


@pytest.mark.parametrize("value", [0.0, 0.5])
def test_blank_and_constant(ctx, value):
    img = np.full((240, 320), value, np.float32)
    k, lv = _compare_levels(ctx, img, 1e-3)
    assert len(k) == 0


def test_batch_equals_single_and_repeat(ctx):
    imgs = [scene(640, 480, seed=1), scene(641, 479, seed=2), scene(150, 120, seed=3), scene(320, 240, seed=4)]
    batch = ctx.akaze_detect(imgs, threshold=1e-4)
    t = ctx.akaze_timing()
    assert t["images"] == 4 and t["kernel_launches"] > 0 and t["keypoints"] == sum(len(b) for b in batch)
    again = ctx.akaze_detect(imgs, threshold=1e-4)
    for i, im in enumerate(imgs):
        one = ctx.akaze_detect([im], threshold=1e-4)[0]
        assert batch[i].tobytes() == one.tobytes() == again[i].tobytes()
        _same_keypoints(batch[i], pa.detect(im, 1e-4))


def test_invalid_input(ctx):
    from regard3d_b200 import capi
    for bad in (np.zeros((2, 50), np.float32), np.zeros((50, 2), np.float32)):
        with pytest.raises(capi.R3DError):
            ctx.akaze_detect([bad])
    img = scene(100, 100, seed=1)
    img[5, 5] = np.nan
    with pytest.raises(capi.R3DError):
        ctx.akaze_detect([img])
    with pytest.raises(capi.R3DError):
        ctx.akaze_detect([scene(100, 100)], diffusivity=0)
    with pytest.raises(capi.R3DError):
        ctx.akaze_detect([scene(100, 100)], threshold=float("inf"))


def test_refine_singular_and_rejected(ctx):
    """The refinement kernel alone: a singular 2x2 system (Dxx = Dyy = -1, Dxy = 1) solves to d = 0 and keeps the
    point; points elsewhere on a random Ldet are refined or rejected; all bit for bit the oracle's."""
    from regard3d_b200 import capi
    rng = np.random.default_rng(5)
    L = rng.normal(size=(40, 48)).astype(np.float32)
    L[9:12, 9:12] = np.float32([[-1.5, 0.5, 0.5], [0.5, 1.0, 0.5], [0.5, 0.5, -1.5]])[::-1]
    kps = np.zeros(1 + 30, pa.keypoint_dtype)
    kps["x"][0], kps["y"][0] = 20.0, 20.0  # ratio 2: pixel (10, 10)
    kps["x"][1:] = rng.integers(1, 47, 30) * 2.0
    kps["y"][1:] = rng.integers(1, 39, 30) * 2.0
    kps["size"], kps["response"], kps["octave"], kps["class_id"] = 4.8, 1.0, 1, 4
    exp = pa.refine(L, 2.0, kps)
    got = ctx.debug_akaze_refine(L, 2.0, kps.view(capi.akaze_keypoint_dtype))
    assert got.tobytes() == exp.tobytes()
    assert got["class_id"][0] == 4 and got["x"][0] == 20.0 and got["y"][0] == 20.0 and got["size"][0] == np.float32(9.6)
    assert (got["class_id"][1:] == -1).any() and (got["class_id"][1:] == 4).any()


def test_image_too_small_for_one_level(ctx):
    """Upstream asserts on an image with no level (2 border + 1 >= a side); here it has no keypoints."""
    from regard3d_b200 import capi
    img = scene(59, 200, seed=1)
    assert len(capi.akaze_levels(59, 200)) == 0
    assert len(ctx.akaze_detect([img])[0]) == 0
    assert len(pa.detect(img)) == 0


def test_two_devices_equal_one():
    import torch
    from regard3d_b200 import capi
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    imgs = [scene(640, 480, seed=s) for s in range(5)]
    c1, c2 = capi.Context((0,)), capi.Context((0, 1))
    try:
        one = c1.akaze_detect(imgs, threshold=1e-4)
        two = c2.akaze_detect(imgs, threshold=1e-4)
        assert c2.akaze_timing()["devices"] == 2
        for a, b in zip(one, two):
            assert a.tobytes() == b.tobytes()
    finally:
        c1.close()
        c2.close()
