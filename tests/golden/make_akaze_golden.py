"""Writes tests/golden/akaze_smoke_v1.npz: one procedural 320x240 gray image and the Fast-AKAZE keypoints the CPU
restatement (oracle/oracle_akaze.cpp) finds in it at threshold 1e-3.  __graft_entry__.smoke() holds the device
detector to them bit for bit.  Records the numpy and (if present) cv2 versions of the machine that wrote it.

    python tests/golden/make_akaze_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.join(HERE, "..", ".."), os.path.join(HERE, "..")]

from akaze_scenes import scene  # noqa: E402
from oracle import pyoracle_akaze as pa  # noqa: E402


def main():
    img = scene(320, 240, seed=2024)
    kps = pa.detect(img, 1e-3)
    try:
        import cv2
        cv = cv2.__version__
    except ImportError:
        cv = "absent"
    out = os.path.join(HERE, "akaze_smoke_v1.npz")
    np.savez_compressed(out, image=img, keypoints=kps.view(np.uint8), threshold=np.float32(1e-3),
                        versions=np.array("numpy %s, cv2 %s" % (np.__version__, cv)))
    print(out, len(kps), "keypoints")


if __name__ == "__main__":
    main()
