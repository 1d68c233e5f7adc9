"""The AKAZE restatement (tests/akaze_cv_ref.py) against live cv2.AKAZE_create(DESCRIPTOR_MLDB, 0, 3, t, 4, 4,
DIFF_PM_G2).detect, the call Regard3D's "AKAZE" detector makes (src/Regard3DFeatures.cpp:578-589).

Bars: the same number of keypoints in the same order; equal class_id, octave and size; response within 1e-5
relative; position within 1e-3 px; angle within 0.01 degrees (mod 360).  The scale space agrees with cv2's only to a
few ulp, so three exceptions are named where they occur:
  - response: a point just above threshold 1e-4 on 641x479 seed 5 is off by 1.21e-5 relative (an absolute error of
    a few ulp of the level's largest response); that case is held to 1.5e-5;
  - position: at levels whose 2x2 refinement system is nearly singular an ulp in Ldet moves the refined point by up
    to 1.13e-3 px (measured: 640x480 seed 21 and 641x479 seed 5 at threshold 1e-4, octave 0); those cases are held
    to 1.5e-3 px;
  - angle: on 640x480 seed 23 at threshold 1e-4 one point (level 7) has two orientation windows whose norms differ in
    the last bits, and cv2 picks the other one (76 degrees apart).
"""
import numpy as np
import pytest

import akaze_cv_ref as ak
from akaze_cv_ref import assert_matches_cv2
from akaze_scenes import scene

cv2 = pytest.importorskip("cv2")

CASES = [(640, 480, s, t) for s in (21, 22, 23) for t in (1e-4, 7e-4, 1e-3)]
CASES += [(641, 479, 5, t) for t in (1e-4, 7e-4, 1e-3)]
CASES += [(150, 120, 3, t) for t in (1e-4, 7e-4, 1e-3)]   # a single octave
CASES += [(100, 100, 4, t) for t in (1e-4, 7e-4, 1e-3)]   # cv2 keeps a fourth level with no interior


def cv2_keypoints(img, threshold):
    det = cv2.AKAZE_create(cv2.AKAZE_DESCRIPTOR_MLDB, 0, 3, threshold, 4, 4, cv2.KAZE_DIFF_PM_G2)
    ref = det.detect(img, None)
    out = np.zeros(len(ref), ak.pa.keypoint_dtype)
    for i, k in enumerate(ref):
        out[i] = (k.pt[0], k.pt[1], k.size, k.angle, k.response, k.octave, k.class_id)
    return out


@pytest.mark.parametrize("w,h,seed,threshold", CASES)
def test_restatement_matches_cv2(w, h, seed, threshold):
    img = scene(w, h, seed=seed)
    assert_matches_cv2(ak.detect(img, threshold), cv2_keypoints(img, threshold), (w, h, seed, threshold))


def test_image_below_one_level():
    img = scene(50, 50, seed=1)
    assert len(ak.detect(img, 1e-4)) == 0 and len(cv2_keypoints(img, 1e-4)) == 0


def test_fast_atan2_deg_against_cv2():
    rng = np.random.default_rng(3)
    y, x = rng.normal(size=(2, 2000)).astype(np.float32)
    y[:4], x[:4] = (0, 0, -1e-9, 1), (1, -1, 1, 0)
    exp = np.float32([cv2.fastAtan2(float(a), float(b)) for a, b in zip(y, x)])
    got = ak.fast_atan2_deg(y, x)
    assert np.abs(got - exp).max() <= 2e-4  # the scalar and the SIMD path of fastAtan32f round differently


def test_passes_change_something():
    _, lv = ak.detect(scene(640, 480, seed=21), 1e-4, levels=True)
    assert any((l["same"] != l["lower"]).any() for l in lv)
    assert any((l["lower"] != l["upper"]).any() for l in lv)
