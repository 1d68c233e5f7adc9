"""Seeded procedural gray images in [0, 1] for the Fast-AKAZE tests and benchmark: overlapping discs, rectangles and
a smooth shading, then a light blur; blob-like structure at several scales gives the detector work on every level."""
import numpy as np


def scene(w, h, seed=0, n_shapes=None):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    img = (0.3 + 0.2 * np.sin(xx / max(w, 1) * 3.0 + rng.uniform(0, 6)) * np.cos(yy / max(h, 1) * 2.0)).astype(np.float32)
    n = n_shapes if n_shapes is not None else max(8, int(w * h / 4000))
    for _ in range(n):
        cx, cy = rng.uniform(0, w), rng.uniform(0, h)
        r = rng.uniform(2, max(3, min(w, h) / 10))
        v = np.float32(rng.uniform(-0.35, 0.35))
        x0, x1 = max(int(cx - r) - 1, 0), min(int(cx + r) + 2, w)
        y0, y1 = max(int(cy - r) - 1, 0), min(int(cy + r) + 2, h)
        if x0 >= x1 or y0 >= y1:
            continue
        sub = (slice(y0, y1), slice(x0, x1))
        if rng.random() < 0.5:
            m = (xx[sub] - cx) ** 2 + (yy[sub] - cy) ** 2 <= r * r
        else:
            m = (np.abs(xx[sub] - cx) <= r) & (np.abs(yy[sub] - cy) <= r * rng.uniform(0.3, 1.0))
        img[sub] += v * m
    img = np.clip(img, 0, 1).astype(np.float32)
    # a 3-tap box blur so edges are not single-pixel steps
    p = np.pad(img, 1, mode="edge")
    img = (p[:-2, 1:-1] + p[1:-1, 1:-1] + p[2:, 1:-1]) / np.float32(3)
    p = np.pad(img, 1, mode="edge")
    img = (p[1:-1, :-2] + p[1:-1, 1:-1] + p[1:-1, 2:]) / np.float32(3)
    return np.ascontiguousarray(img, np.float32)
