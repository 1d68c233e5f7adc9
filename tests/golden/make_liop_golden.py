#!/usr/bin/env python
"""Generate the LIOP golden fixtures (run in the BUILD CONTAINER, where /root/reference and cv2 exist):

    python tests/golden/make_liop_golden.py

  liop_ref_v1.npz        patches (float32 41x41, seeded: smooth / noisy / quantised-with-ties / flat / steps) and the
                         descriptors THE REFERENCE ITSELF computes for them: oracle/_ref/libvlliop_ref.so, built by
                         oracle/Makefile from /root/reference/src/thirdparty/liop/vl_liop.c (r3d_vl_liopdesc_process).
  liop_ref_mixed_v1.npz  the reference's descriptors of mixed_patches() (noise, quantised with ties, row sums).
  liop_patch_cv2_v1.npz  a seeded image, keypoints, and the 41x41 patches cv2 (version recorded) produces with the
                         reference's call sequence (src/Regard3DFeatures.cpp:766-806): warpAffine(INTER_LINEAR |
                         WARP_INVERSE_MAP) then GaussianBlur(sigma = 1.2); warped-only patches are stored too.
The GPU box has neither the reference tree nor a reason to trust cv2's CPU dispatch: tests there read these files."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from oracle import pyoracle as po  # noqa: E402


def make_patches(seed=20260924):
    rng = np.random.default_rng(seed)
    out = []
    yy, xx = np.mgrid[0:41, 0:41].astype(np.float32)
    for k in range(24):                                   # smooth random fields
        f = rng.standard_normal((41, 41)).astype(np.float32)
        import cv2
        out.append(cv2.GaussianBlur(f, (0, 0), 1.0 + 0.2 * k))
    for k in range(16):                                   # raw noise
        out.append(rng.random((41, 41)).astype(np.float32))
    for k in range(24):                                   # quantised: many exact ties in the intensity order
        q = [2, 3, 4, 8, 16, 64][k % 6]
        out.append((np.floor(rng.random((41, 41)) * q) / q).astype(np.float32))
    for k in range(8):                                    # piecewise constant (polygon-like) regions
        a, b, c = rng.standard_normal(3)
        out.append(((a * (xx - 20) + b * (yy - 20) + 3 * c) > 0).astype(np.float32) * np.float32(rng.random()) + np.float32(0.1 * k))
    out.append(np.zeros((41, 41), np.float32))            # flat (all keys equal: the quick sort's worst case)
    out.append(np.full((41, 41), 0.7, np.float32))
    out.append((xx / 40).astype(np.float32))              # ramps
    out.append((yy / 40).astype(np.float32))
    out.append(((xx + yy) % 2).astype(np.float32))        # checkerboard
    return np.stack(out).astype(np.float32)


def mixed_patches(seed=11):
    rng = np.random.default_rng(seed)
    patches = []
    for k in range(120):
        p = rng.random((41, 41)).astype(np.float32)
        if k % 3 == 1:
            p = np.floor(p * (2 + k % 7)) / (2 + k % 7)        # exact ties: the order is the quick sort's own
        if k % 3 == 2:
            p = np.cumsum(p, 1) / 41
        patches.append(p.astype(np.float32))
    return np.stack(patches)


def main():
    import cv2
    assert po.liop_ref_available(), "needs /root/reference (oracle/_ref)"
    patches = make_patches()
    desc = po.liop_ref_process(patches)
    np.savez_compressed(os.path.join(HERE, "liop_ref_v1.npz"), patches=patches, desc=desc,
                        source="r3d_vl_liopdesc_process of /root/reference/src/thirdparty/liop/vl_liop.c (oracle/_ref)")
    np.savez_compressed(os.path.join(HERE, "liop_ref_mixed_v1.npz"), desc=po.liop_ref_process(mixed_patches()),
                        source="r3d_vl_liopdesc_process of src/thirdparty/liop/vl_liop.c (oracle/_ref)")
    # ---- OpenCV patch extraction ----
    rng = np.random.default_rng(20260925)
    h, w = 240, 320
    img = cv2.GaussianBlur(rng.random((h, w)).astype(np.float32), (0, 0), 2.0)
    img += 0.3 * (np.add.outer(np.arange(h), np.arange(w)) % 37 < 18)
    img = img.astype(np.float32)
    n = 96
    kps = np.stack([rng.uniform(-5, w + 5, n), rng.uniform(-5, h + 5, n), rng.uniform(4, 60, n), rng.uniform(0, 360, n)], 1).astype(np.float32)
    kps[0] = (160.0, 120.0, 41.0, 270.0)                 # identity-like map
    kps[1] = (0.0, 0.0, 20.0, 0.0)                       # corner: constant border
    factor = np.float32(2.5)
    warped, blurred = [], []
    for x, y, size, angle in kps:
        M = po.liop_affine(x, y, size, angle, factor)    # the float arithmetic of Regard3DFeatures.cpp:773-800
        p = cv2.warpAffine(img, M, (41, 41), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP)
        warped.append(p.copy())
        blurred.append(cv2.GaussianBlur(p, (0, 0), 1.2))
    keep = 40                                            # the first keypoints only: the file stays below 1 MB
    np.savez_compressed(os.path.join(HERE, "liop_patch_cv2_v1.npz"), img=img, kps=kps[:keep], factor=factor,
                        warped=np.stack(warped[:keep]), blurred=np.stack(blurred[:keep]), cv2_version=cv2.__version__,
                        gauss_kernel=cv2.getGaussianKernel(11, 1.2, cv2.CV_32F).ravel())
    print("wrote liop_ref_v1.npz (%d patches) and liop_patch_cv2_v1.npz (%d keypoints), cv2 %s" % (len(patches), keep, cv2.__version__))


if __name__ == "__main__":
    main()
