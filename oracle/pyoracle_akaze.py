"""ctypes wrapper of the CPU ORACLE of the Fast-AKAZE detector (oracle/_build/liboracle_akaze.so, oracle/akaze.mk).

TEST INFRASTRUCTURE ONLY, like pyoracle: importable from tests/, __graft_entry__.smoke() and scripts/bench_akaze.py.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liboracle_akaze.so")

level_dtype = np.dtype([("octave", np.int32), ("sublevel", np.int32), ("width", np.int32), ("height", np.int32),
                        ("sigma_size", np.int32), ("border", np.int32), ("esigma", np.float32), ("etime", np.float32),
                        ("ratio", np.float32), ("n_tau", np.uint32)])
# the same layout as r3d_akaze_keypoint: angle in degrees after Regard3D's conversion (-1 for candidates)
keypoint_dtype = np.dtype([("x", np.float32), ("y", np.float32), ("size", np.float32), ("angle", np.float32),
                           ("response", np.float32), ("octave", np.int32), ("class_id", np.int32)])
ARRAYS = ("Lt", "Lsmooth", "Lx", "Ly", "Ldet")


def build(force=False):
    """Compile liboracle_akaze.so with oracle/akaze.mk."""
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "akaze.mk"] + (["-B"] if force else []))
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_akaze_detect.restype = C.c_void_p
        v, i = C.c_void_p, C.c_int
        for f, args in (("orc_akaze_free", [v]), ("orc_akaze_num_levels", [v]), ("orc_akaze_get_level", [v, i, v]),
                        ("orc_akaze_get_kcontrast", [v, i]), ("orc_akaze_get_array", [v, i, i, v]),
                        ("orc_akaze_num_candidates", [v, i]), ("orc_akaze_get_candidates", [v, i, v, v, v]),
                        ("orc_akaze_num_keypoints", [v]), ("orc_akaze_get_keypoints", [v, v, v]),
                        ("orc_akaze_get_stats", [v, v])):
            getattr(_lib, f).argtypes = args
        _lib.orc_akaze_get_kcontrast.restype = C.c_float
        _lib.orc_akaze_k_percentile.restype = C.c_float
        _lib.orc_akaze_angle.restype = C.c_float
        _lib.orc_akaze_angle.argtypes = [C.c_float, C.c_float]
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def level_table(w, h, octaves=4, sublevels=4):
    out = np.zeros(64, level_dtype)
    n = lib().orc_akaze_level_table(C.c_int(w), C.c_int(h), C.c_int(octaves), C.c_int(sublevels), _p(out), C.c_int(64))
    return out[:n].copy()


def fed_tau(T, tau_max=0.25):
    out = np.zeros(4096, np.float32)
    n = lib().orc_akaze_fed_tau(C.c_float(T), C.c_float(tau_max), _p(out), C.c_int(len(out)))
    return out[:n].copy()


def gaussian_kernel(n, sigma):
    k = np.zeros(n, np.float32)
    lib().orc_akaze_gaussian_kernel(C.c_int(n), C.c_double(sigma), _p(k))
    return k


def deriv_kernels(dx, dy, scale):
    kx = np.zeros(64, np.float32)
    ky = np.zeros(64, np.float32)
    n = lib().orc_akaze_deriv_kernels(C.c_int(dx), C.c_int(dy), C.c_int(scale), _p(kx), _p(ky))
    return kx[:n].copy(), ky[:n].copy()


def gaussian_blur(img, sigma):
    img = _f32(img)
    out = np.zeros_like(img)
    lib().orc_akaze_gaussian_blur(_p(img), C.c_int(img.shape[1]), C.c_int(img.shape[0]), C.c_float(sigma), _p(out))
    return out


def scharr(img, dx, dy):
    img = _f32(img)
    out = np.zeros_like(img)
    lib().orc_akaze_scharr(_p(img), C.c_int(img.shape[1]), C.c_int(img.shape[0]), C.c_int(dx), C.c_int(dy), _p(out))
    return out


def sep_filter(img, kx, ky):
    img, kx, ky = _f32(img), _f32(kx), _f32(ky)
    out = np.zeros_like(img)
    lib().orc_akaze_sep_filter(_p(img), C.c_int(img.shape[1]), C.c_int(img.shape[0]), _p(kx), C.c_int(len(kx)), _p(ky),
                               C.c_int(len(ky)), _p(out))
    return out


def halfsample(img):
    img = _f32(img)
    out = np.zeros((img.shape[0] // 2, img.shape[1] // 2), np.float32)
    lib().orc_akaze_halfsample(_p(img), C.c_int(img.shape[1]), C.c_int(img.shape[0]), _p(out))
    return out


def fast_atan2(y, x):
    y, x = _f32(y), _f32(x)
    out = np.zeros_like(y)
    lib().orc_akaze_fast_atan2(_p(y), _p(x), C.c_int(y.size), _p(out))
    return out


def solve2(A, b):
    A, b = _f32(A), _f32(b)
    x = np.zeros(2, np.float32)
    lib().orc_akaze_solve2(_p(A), _p(b), _p(x))
    return x


def k_percentile(lx, ly, perc=0.7, nbins=300):
    lx, ly = _f32(lx), _f32(ly)
    return lib().orc_akaze_k_percentile(_p(lx), _p(ly), C.c_int(lx.shape[1]), C.c_int(lx.shape[0]), C.c_float(perc),
                                        C.c_int(nbins))


def gauss25():
    g = np.zeros((7, 7), np.float32)
    lib().orc_akaze_gauss25(_p(g))
    return g


def angle(max_x, max_y):
    return lib().orc_akaze_angle(C.c_float(max_x), C.c_float(max_y))


def refine(ldet, ratio, kps):
    """Subpixel refinement alone on points (keypoint_dtype) of one level's Ldet; rejected points get class_id -1."""
    ldet = _f32(ldet)
    kps = np.ascontiguousarray(kps, keypoint_dtype)
    out = np.zeros_like(kps)
    lib().orc_akaze_refine(_p(ldet), C.c_int(ldet.shape[1]), C.c_float(ratio), _p(kps), C.c_int(len(kps)), _p(out))
    return out


def detect(img, threshold=0.001, octaves=4, sublevels=4, levels=False, stats=None):
    """The detector on one float32 gray image in [0, 1].  Returns the keypoints (keypoint_dtype) and, with
    levels=True, also a list of per-level dicts: the level record, kcontrast, the five arrays, the candidates after
    the same-level pass and their deletion flags after the lower- and the upper-level pass.  stats: a dict that
    receives how often the rarer branches ran ("replaced", "singular", "rejected")."""
    img = _f32(img)
    h, w = img.shape
    L = lib()
    s = L.orc_akaze_detect(_p(img), C.c_int(w), C.c_int(h), C.c_float(threshold), C.c_int(octaves), C.c_int(sublevels))
    try:
        n = L.orc_akaze_num_keypoints(s)
        kps = np.zeros(n, keypoint_dtype)
        ori = np.zeros((n, 2), np.float32)
        L.orc_akaze_get_keypoints(s, _p(kps), _p(ori))
        if stats is not None:
            st = np.zeros(3, np.int32)
            L.orc_akaze_get_stats(s, _p(st))
            stats.update(replaced=int(st[0]), singular=int(st[1]), rejected=int(st[2]))
        if not levels:
            return kps
        out = []
        for i in range(L.orc_akaze_num_levels(s)):
            rec = np.zeros(1, level_dtype)
            L.orc_akaze_get_level(s, i, _p(rec))
            lw, lh = int(rec["width"][0]), int(rec["height"][0])
            d = {"level": rec[0], "kcontrast": L.orc_akaze_get_kcontrast(s, i)}
            for k, name in enumerate(ARRAYS):
                a = np.zeros((lh, lw), np.float32)
                L.orc_akaze_get_array(s, i, k, _p(a))
                d[name] = a
            nc = L.orc_akaze_num_candidates(s, i)
            c = np.zeros(nc, keypoint_dtype)
            dl = np.zeros(nc, np.uint8)
            du = np.zeros(nc, np.uint8)
            L.orc_akaze_get_candidates(s, i, _p(c), _p(dl), _p(du))
            d.update(candidates=c, deleted_lower=dl.astype(bool), deleted_upper=du.astype(bool))
            out.append(d)
        return kps, out, ori
    finally:
        L.orc_akaze_free(s)
