"""ctypes wrapper of the CPU ORACLE of the resection step (oracle/_build/liboracle_resection.so, oracle/resection.mk).

TEST INFRASTRUCTURE ONLY, like pyoracle: importable from tests/, __graft_entry__.smoke() and scripts/bench_resection.py.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.pyoracle import BAOptions, _p, default_ba_options

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liboracle_resection.so")


def build(force=False):
    """Compile liboracle_resection.so (and liboracle.so, which it links) with oracle/resection.mk."""
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "resection.mk"] + (["-B"] if force else []))
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
    return _lib


RESECT_OK, RESECT_TOO_FEW, RESECT_NO_INTRINSIC, RESECT_NO_MODEL = 0, 1, 2, 3
resection_dtype = np.dtype([
    ("view_id", np.uint32), ("status", np.int32), ("n_inliers", np.uint32), ("found_residual_precision", np.float64),
    ("rotation", np.float64, (3, 3)), ("center", np.float64, 3), ("translation", np.float64, 3),
    ("rotation_ransac", np.float64, (3, 3)), ("translation_ransac", np.float64, 3), ("lm_iterations", np.uint32),
    ("lm_successful_steps", np.uint32), ("lm_termination", np.int32), ("lm_initial_cost", np.float64),
    ("lm_final_cost", np.float64)], align=True)


class ResectionOptions(C.Structure):
    _fields_ = [("precision_px", C.c_double), ("max_iter", C.c_uint32), ("refine", C.c_int), ("ba", BAOptions)]


class BASummary(C.Structure):
    _fields_ = [("iterations", C.c_uint32), ("successful_steps", C.c_uint32), ("initial_cost", C.c_double),
                ("final_cost", C.c_double), ("termination", C.c_int), ("seconds_total", C.c_double),
                ("seconds_linear", C.c_double)]


def resection_options(precision_px=float("inf"), max_iter=4096, refine=True, **ba):
    o = ResectionOptions()
    o.precision_px = precision_px
    o.max_iter = max_iter
    o.refine = int(refine)
    o.ba = default_ba_options(refine_intrinsics=0, n_threads=1)
    for k, v in ba.items():
        setattr(o.ba, k, v)
    return o


def intr8(focal, ppx, ppy, disto=()):
    a = np.zeros(8)
    a[:3] = focal, ppx, ppy
    a[3:3 + len(disto)] = disto
    return a


def p3p(K, X, x):
    """One sample: the models K [R | t] (n x 3 x 4) in the order the AC-RANSAC tries them."""
    P = np.zeros((4, 3, 4))
    n = lib().orc_p3p(_p(np.ascontiguousarray(K, np.float64)), _p(np.ascontiguousarray(X, np.float64)),
                      _p(np.ascontiguousarray(x, np.float64)), _p(P))
    return P[:n].copy()


def undistort(model, intr, xy):
    xy = np.ascontiguousarray(xy, np.float64)
    out = np.zeros_like(xy)
    lib().orc_undistort(C.c_int(model), _p(np.ascontiguousarray(intr, np.float64)), _p(xy), C.c_uint32(len(xy)), _p(out))
    return out


def refine(model, intr, X, x, pose, **ba):
    """Pose-only LM from `pose` (angle-axis | t): (refined pose, summary dict)."""
    X = np.ascontiguousarray(X, np.float64)
    x = np.ascontiguousarray(x, np.float64)
    pose = np.array(pose, np.float64)
    o = default_ba_options(refine_intrinsics=0, n_threads=1)
    for k, v in ba.items():
        setattr(o, k, v)
    s = BASummary()
    lib().orc_resect_refine(C.c_int(model), _p(np.ascontiguousarray(intr, np.float64)), _p(X), _p(x), C.c_uint32(len(X)),
                            C.byref(o), _p(pose), C.byref(s))
    return pose, {k: getattr(s, k) for k, _ in BASummary._fields_}


def resect_view(X, x, width, height, model, intr, **opts):
    """One view: (result record, AC-RANSAC inlier indices in residual order)."""
    X = np.ascontiguousarray(X, np.float64)
    x = np.ascontiguousarray(x, np.float64)
    M = len(X)
    r = np.zeros(1, resection_dtype)
    inl = np.zeros(max(M, 1), np.uint32)
    o = resection_options(**opts)
    lib().orc_resect_view(_p(X), _p(x), C.c_uint32(M), C.c_uint32(width), C.c_uint32(height), C.c_int(model),
                          _p(np.ascontiguousarray(intr, np.float64)), C.byref(o), _p(r), _p(inl))
    return r[0], inl[:int(r[0]["n_inliers"])].copy()


def resect_views(first, count, widths, heights, models, intrs, X, x, n_threads=0, **opts):
    """orc_resect_views over a batch: (records[n], inlier ofs[n + 1], inlier indices)."""
    first = np.ascontiguousarray(first, np.uint64)
    count = np.ascontiguousarray(count, np.uint64)
    n = len(first)
    X = np.ascontiguousarray(X, np.float64)
    x = np.ascontiguousarray(x, np.float64)
    out = np.zeros(n, resection_dtype)
    inl = np.zeros(max(1, len(x)), np.uint32)
    ofs = np.zeros(n + 1, np.uint64)
    o = resection_options(**opts)
    lib().orc_resect_views(C.c_uint32(n), _p(first), _p(count), _p(np.ascontiguousarray(widths, np.uint32)),
                           _p(np.ascontiguousarray(heights, np.uint32)), _p(np.ascontiguousarray(models, np.int32)),
                           _p(np.ascontiguousarray(intrs, np.float64)), _p(X), _p(x), C.byref(o), _p(out), _p(inl), _p(ofs),
                           C.c_int(n_threads))
    return out, ofs, inl[:int(ofs[n])].copy()
