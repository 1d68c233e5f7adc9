"""Write tests/golden/akaze_cv_v1.npz: cv2.AKAZE_create(DESCRIPTOR_MLDB, 0, 3, t, 4, 4, DIFF_PM_G2).detect's keypoints
on procedural scenes (tests/akaze_scenes.py, regenerated from their seeds), so the GPU tests can hold the device to
cv2 on a machine without cv2.  Run from the repository root: python tests/golden/make_akaze_cv_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

import cv2  # noqa: E402

from akaze_scenes import scene  # noqa: E402
from test_oracle_akaze_cv import cv2_keypoints  # noqa: E402

CASES = [(640, 480, 21, 7e-4), (640, 480, 22, 1e-3), (641, 479, 5, 7e-4), (150, 120, 3, 1e-4)]

if __name__ == "__main__":
    out = {"cases": np.array(CASES, np.float64), "cv2_version": np.array(cv2.__version__),
           "numpy_version": np.array(np.__version__)}
    for k, (w, h, seed, t) in enumerate(CASES):
        out["kps%d" % k] = cv2_keypoints(scene(w, h, seed=seed), t)
    np.savez_compressed(os.path.join(HERE, "akaze_cv_v1.npz"), **out)
