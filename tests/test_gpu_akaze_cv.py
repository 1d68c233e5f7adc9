"""-m gpu: R3D_DETECTOR_AKAZE (OpenCV 4's cv::AKAZE::detect, Regard3D's "AKAZE") on the device against the CPU
restatement (tests/akaze_cv_ref.py): every level's arrays, the masks after each of the three passes and every keypoint
field, bit for bit; against cv2's own keypoints stored in tests/golden/akaze_cv_v1.npz; and through feature
extraction, against LIOP of the restatement's keypoints."""
import os

import numpy as np
import pytest

import akaze_cv_ref as ak
import features_ref as fr
from akaze_scenes import scene
from oracle import pyoracle as po
from oracle import pyoracle_akaze as pa

pytestmark = pytest.mark.gpu

AKAZE = 1
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "akaze_cv_v1.npz")


@pytest.fixture(scope="module")
def ctx():
    from regard3d_b200 import capi
    c = capi.Context((0,))
    yield c
    c.close()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _compare(ctx, img, threshold):
    exp_k, exp_l = ak.detect(img, threshold, levels=True)
    got_l = ctx.debug_akaze_masks(img, threshold=threshold)
    assert len(got_l) == len(exp_l)
    for i, (g, e) in enumerate(zip(got_l, exp_l)):
        assert g["level"].tobytes() == e["level"].tobytes(), "level %d record" % i
        for name in pa.ARRAYS:
            assert np.array_equal(_bits(g[name]), _bits(e[name])), "level %d %s differs" % (i, name)
        for name in ("same", "lower", "upper"):
            assert np.array_equal(g[name], e[name]), "level %d mask after the %s pass" % (i, name)
    got_k = ctx.akaze_detect([img], detector=AKAZE, threshold=threshold)[0]
    assert len(got_k) == len(exp_k)
    assert got_k.tobytes() == exp_k.tobytes(), "keypoints differ from the restatement's"
    return exp_k, exp_l


@pytest.mark.parametrize("w,h,threshold", [
    (640, 480, 7e-4),
    (641, 479, 1e-3),     # odd sides
    (150, 120, 1e-4),     # one octave
    (100, 100, 1e-4),     # the level list ends mid-octave
    (640, 480, 1e-4),
    (640, 480, 1e-2),
])
def test_levels_masks_and_keypoints_bit_identical(ctx, w, h, threshold):
    k, lv = _compare(ctx, scene(w, h, seed=w + h), threshold)
    if (w, h, threshold) == (640, 480, 1e-4):
        # every pass changes something on this scene
        assert any((l["same"] != l["lower"]).any() for l in lv)
        assert any((l["lower"] != l["upper"]).any() for l in lv)
        assert len(k) > 100


def test_large_image(ctx):
    _compare(ctx, scene(4000, 3000, seed=7), 1e-3)


@pytest.mark.parametrize("value", [0.0, 0.5])
def test_blank_and_constant(ctx, value):
    k, _ = _compare(ctx, np.full((240, 320), value, np.float32), 1e-3)
    assert len(k) == 0


def test_batch_equals_single_and_repeat(ctx):
    imgs = [scene(640, 480, seed=1), scene(641, 479, seed=2), scene(150, 120, seed=3), scene(59, 200, seed=4),
            scene(320, 240, seed=5)]
    batch = ctx.akaze_detect(imgs, detector=AKAZE, threshold=1e-4)
    assert ctx.akaze_timing()["keypoints"] == sum(len(b) for b in batch)
    again = ctx.akaze_detect(imgs, detector=AKAZE, threshold=1e-4)
    for i, im in enumerate(imgs):
        one = ctx.akaze_detect([im], detector=AKAZE, threshold=1e-4)[0]
        assert batch[i].tobytes() == one.tobytes() == again[i].tobytes()
        assert one.tobytes() == ak.detect(im, 1e-4).tobytes()
    assert len(batch[3]) == 0  # no level


def test_two_devices_equal_one():
    import torch
    from regard3d_b200 import capi
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    imgs = [scene(640, 480, seed=s) for s in range(5)]
    c1, c2 = capi.Context((0,)), capi.Context((0, 1))
    try:
        one = c1.akaze_detect(imgs, detector=AKAZE, threshold=1e-4)
        two = c2.akaze_detect(imgs, detector=AKAZE, threshold=1e-4)
        assert c2.akaze_timing()["devices"] == 2
        for a, b in zip(one, two):
            assert a.tobytes() == b.tobytes()
    finally:
        c1.close()
        c2.close()


def test_golden_cv2_keypoints(ctx):
    """The device against cv2.AKAZE_create(...).detect's own keypoints, recorded by make_akaze_cv_golden.py, within
    the bounds of tests/test_oracle_akaze_cv.py."""
    g = np.load(GOLDEN)
    for k, (w, h, seed, thr) in enumerate(g["cases"]):
        got = ctx.akaze_detect([scene(int(w), int(h), seed=int(seed))], detector=AKAZE, threshold=float(thr))[0]
        exp = g["kps%d" % k]
        ak.assert_matches_cv2(got, exp, (int(w), int(h), int(seed), float(thr)))


@pytest.mark.parametrize("w,h,threshold", [(640, 480, 7e-4), (641, 479, 1e-4), (4000, 3000, 1e-3)])
def test_extract_features_akaze(ctx, tmp_path, w, h, threshold):
    """AKAZE keypoints described with LIOP (size factor 8) at their cv::AKAZE angle: descriptors bit for bit LIOP of
    the restatement's keypoints, files byte for byte the OpenMVG writers'."""
    img = scene(w, h, seed=w + h)
    gpu, ref = tmp_path / "gpu", tmp_path / "ref"
    gpu.mkdir()
    ref.mkdir()
    got_k, got_d = ctx.extract_features([img], out_dir=str(gpu), basenames=["im"], threshold=threshold,
                                        detector=AKAZE)[0]
    exp_k = ak.detect(img, threshold)
    k4 = np.stack([exp_k["x"], exp_k["y"], exp_k["size"], exp_k["angle"]], 1).astype(np.float32)
    exp_d = po.liop_describe(img, k4, 8.0)
    fr.write(ref, "im", exp_k, exp_d)
    assert got_k.tobytes() == exp_k.tobytes()
    assert np.array_equal(_bits(got_d), _bits(exp_d))
    for ext in (".feat", ".desc"):
        assert open(str(gpu / ("im" + ext)), "rb").read() == open(str(ref / ("im" + ext)), "rb").read()


def test_fast_akaze_through_the_new_calls_equals_the_old(ctx):
    from regard3d_b200 import capi
    imgs = [scene(640, 480, seed=3), scene(641, 479, seed=4)]
    old = ctx.akaze_detect(imgs, threshold=1e-4)
    new = ctx.akaze_detect(imgs, detector=capi.DETECTOR_FAST_AKAZE, threshold=1e-4)
    for a, b in zip(old, new):
        assert a.tobytes() == b.tobytes()
    old_x = ctx.extract_features(imgs, threshold=1e-4)
    new_x = ctx.extract_features(imgs, threshold=1e-4, detector=capi.DETECTOR_FAST_AKAZE)
    for (ka, da), (kb, db) in zip(old_x, new_x):
        assert ka.tobytes() == kb.tobytes() and np.array_equal(_bits(da), _bits(db))
    # the two detectors differ: AKAZE places octave >= 1 points half a level pixel further, and angles differ
    ak_k = ctx.akaze_detect(imgs[:1], detector=AKAZE, threshold=1e-4)[0]
    assert ak_k.tobytes() != old[0].tobytes()


def test_invalid_input(ctx):
    from regard3d_b200 import capi
    for bad in (np.zeros((2, 50), np.float32), np.zeros((50, 2), np.float32)):
        with pytest.raises(capi.R3DError):
            ctx.akaze_detect([bad], detector=AKAZE)
    img = scene(100, 100, seed=1)
    img[5, 5] = np.nan
    with pytest.raises(capi.R3DError):
        ctx.akaze_detect([img], detector=AKAZE)
    with pytest.raises(capi.R3DError):
        ctx.akaze_detect([scene(100, 100)], detector=AKAZE, diffusivity=0)
    with pytest.raises(capi.R3DError):
        ctx.akaze_detect([scene(100, 100)], detector=AKAZE, threshold=float("inf"))
    for det in (-1, 2):
        with pytest.raises(capi.R3DError):
            ctx.akaze_detect([scene(100, 100)], detector=det)
        with pytest.raises(capi.R3DError):
            ctx.extract_features([scene(100, 100)], detector=det)
