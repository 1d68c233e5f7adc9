"""ctypes wrapper of the CPU ORACLE of the relative-pose step (oracle/_build/liboracle_relpose.so, oracle/relpose.mk).

TEST INFRASTRUCTURE ONLY, like pyoracle: importable from tests/, __graft_entry__.smoke() and scripts/bench_relpose.py.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.pyoracle import BAOptions, _p, _ptr_array, default_ba_options, indmatch_dtype

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liboracle_relpose.so")


def build(force=False):
    """Compile liboracle_relpose.so (and liboracle.so, which it links) with oracle/relpose.mk."""
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "relpose.mk"] + (["-B"] if force else []))
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_relative_poses.restype = C.c_int64
    return _lib


RELPOSE_OK, RELPOSE_TOO_FEW, RELPOSE_NO_INTRINSIC, RELPOSE_NO_MODEL, RELPOSE_CHEIRALITY = 0, 1, 2, 3, 4
relpose_dtype = np.dtype([
    ("I", np.uint32), ("J", np.uint32), ("status", np.int32), ("n_inliers", np.uint32),
    ("found_residual_precision", np.float64), ("E", np.float64, (3, 3)), ("rotation", np.float64, (3, 3)),
    ("translation", np.float64, 3), ("ba_iterations", np.uint32), ("ba_successful_steps", np.uint32),
    ("ba_termination", np.int32), ("ba_initial_cost", np.float64), ("ba_final_cost", np.float64)], align=True)


class RelposeOptions(C.Structure):
    _fields_ = [("precision_px", C.c_double), ("max_iter", C.c_uint32), ("refine", C.c_int), ("ba", BAOptions)]


def relpose_options(precision_px=2.5, max_iter=256, refine=True, **ba):
    o = RelposeOptions()
    o.precision_px = precision_px
    o.max_iter = max_iter
    o.refine = int(refine)
    o.ba = default_ba_options(refine_intrinsics=0, n_threads=1)
    for k, v in ba.items():
        setattr(o.ba, k, v)
    return o


def motions_from_essential(E):
    """MotionFromEssential: (Rs[4,3,3], ts[4,3])."""
    E = np.ascontiguousarray(E, np.float64)
    Rs = np.zeros((4, 3, 3))
    ts = np.zeros((4, 3))
    lib().orc_motions_from_essential(_p(E), _p(Rs), _p(ts))
    return Rs, ts


def relative_pose(xI, xJ, wI, hI, wJ, hJ, Kpair, **opts):
    """One pair: (result record, AC-RANSAC inlier indices in residual order)."""
    xI = np.ascontiguousarray(xI, np.float64)
    xJ = np.ascontiguousarray(xJ, np.float64)
    Kpair = np.ascontiguousarray(Kpair, np.float64)
    M = xI.shape[0]
    r = np.zeros(1, relpose_dtype)
    inl = np.zeros(max(M, 1), np.uint32)
    o = relpose_options(**opts)
    lib().orc_relative_pose(_p(xI), _p(xJ), C.c_uint32(M), C.c_uint32(wI), C.c_uint32(hI), C.c_uint32(wJ), C.c_uint32(hJ),
                            _p(Kpair), C.byref(o), _p(r), _p(inl))
    return r[0], inl[:int(r[0]["n_inliers"])].copy()


def relative_poses(xys, widths, heights, Ks, pairs, put_ofs, put, n_threads=0, **opts):
    """orc_relative_poses over a pair CSR: (records[P], inlier ofs[P+1], inlier matches)."""
    xys = [np.ascontiguousarray(x, np.float32) for x in xys]
    pairs = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
    P = pairs.shape[0]
    widths = np.ascontiguousarray(widths, np.uint32)
    heights = np.ascontiguousarray(heights, np.uint32)
    Ks = np.ascontiguousarray(Ks, np.float64)
    put_ofs = np.ascontiguousarray(put_ofs, np.uint64)
    put = np.ascontiguousarray(put, indmatch_dtype)
    out = np.zeros(P, relpose_dtype)
    inl = np.zeros(max(1, put.shape[0]), indmatch_dtype)
    inl_ofs = np.zeros(P + 1, np.uint64)
    o = relpose_options(**opts)
    fn = lib().orc_relative_poses
    n = fn(_ptr_array(xys), _p(widths), _p(heights), _p(Ks), C.c_uint32(len(xys)), _p(pairs), C.c_uint64(P), _p(put_ofs),
           _p(put), C.byref(o), _p(out), _p(inl_ofs), _p(inl), C.c_int(n_threads))
    return out, inl_ofs, inl[:n].copy()
