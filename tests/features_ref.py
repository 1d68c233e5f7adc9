"""CPU reference of the feature stage, composed from the oracle: Fast-AKAZE (oracle/oracle_akaze.cpp), LIOP-144 with
Regard3D's size factor 8 (oracle/oracle_liop.cpp), then OpenMVG's .feat / .desc writers (oracle/oracle_io.cpp)."""
import os

import numpy as np

from oracle import pyoracle as po
from oracle import pyoracle_akaze as pa


def xyso(kps):
    """SIOPointFeature of each keypoint: x, y, scale = size / 2, orientation (degrees)."""
    return np.ascontiguousarray(np.stack([kps["x"], kps["y"], kps["size"] / np.float32(2), kps["angle"]], 1), np.float32)


def extract(img, threshold=1e-3, factor=8.0):
    """(keypoints in upstream order, (n, 144) descriptors) of one float gray image."""
    kps = pa.detect(img, threshold)
    if len(kps) == 0:
        return kps, np.zeros((0, 144), np.float32)
    k4 = np.stack([kps["x"], kps["y"], kps["size"], kps["angle"]], 1).astype(np.float32)
    return kps, po.liop_describe(img, k4, factor)


def write(out_dir, basename, kps, desc):
    base = os.path.join(str(out_dir), basename)
    assert po.save_feat(base + ".feat", xyso(kps)) == 0
    assert po.save_desc(base + ".desc", np.ascontiguousarray(desc, np.float32).reshape(-1, 144)) == 0


def extract_to(out_dir, images, basenames, threshold=1e-3):
    out = []
    for img, name in zip(images, basenames):
        k, d = extract(img, threshold)
        write(out_dir, name, k, d)
        out.append((k, d))
    return out
