"""ctypes wrapper of the CPU ORACLE of the colour plan, the coloured PLY and the undistortion
(oracle/_build/liboracle_export.so, oracle/export.mk).

TEST INFRASTRUCTURE ONLY, like pyoracle: importable from tests/ and scripts/bench_export.py.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.pyoracle import _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liboracle_export.so")


def build(force=False):
    """Compile liboracle_export.so with oracle/export.mk."""
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "export.mk"] + (["-B"] if force else []))
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_undistort_image.argtypes = [C.c_int, C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_void_p,
                                             C.c_uint32, C.c_uint32, C.c_void_p]
        _lib.orc_write_colorized_ply.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_char_p]
    return _lib


class OracleError(RuntimeError):
    def __init__(self, what):
        super().__init__("oracle %s rejected its input" % what)


def flatten(views, landmarks):
    """views: dicts with id_view / width / height (SfmData.views()); landmarks: dicts with id / X / obs
    (SfmData.landmarks()), obs as (id_view, id_feat, x, y).  -> the arrays orc_colorize_plan reads."""
    vid = np.array([v["id_view"] for v in views], np.uint32)
    vw = np.array([v["width"] for v in views], np.uint32)
    vh = np.array([v["height"] for v in views], np.uint32)
    lms = sorted(landmarks, key=lambda l: l["id"])
    lid = np.array([l["id"] for l in lms], np.uint32)
    ofs = np.zeros(len(lms) + 1, np.uint64)
    ofs[1:] = np.cumsum([len(l["obs"]) for l in lms])
    ov = np.array([o[0] for l in lms for o in l["obs"]], np.uint32)
    oxy = np.array([(o[2], o[3]) for l in lms for o in l["obs"]], np.float64).reshape(-1, 2)
    return vid, vw, vh, lid, ofs, ov, oxy


def colorize_plan(view_ids, widths, heights, lm_ids, obs_ofs, obs_view, obs_xy):
    """orc_colorize_plan: (round_view[:n_rounds], lm_round, lm_pixel (n_lm, 2) as (x, y)); OracleError when rejected."""
    arrs = [np.ascontiguousarray(a, t) for a, t in ((view_ids, np.uint32), (widths, np.uint32), (heights, np.uint32),
                                                     (lm_ids, np.uint32), (obs_ofs, np.uint64), (obs_view, np.uint32),
                                                     (obs_xy, np.float64))]
    nv, nl = len(arrs[0]), len(arrs[3])
    rv = np.zeros(max(nv, 1), np.uint32)
    nr = C.c_uint32()
    lr = np.zeros(max(nl, 1), np.uint32)
    lp = np.zeros((max(nl, 1), 2), np.int32)
    rc = lib().orc_colorize_plan(C.c_uint32(nv), _p(arrs[0]), _p(arrs[1]), _p(arrs[2]), C.c_uint32(nl), _p(arrs[3]),
                                 _p(arrs[4]), _p(arrs[5]), _p(arrs[6]), _p(rv), C.byref(nr), _p(lr), _p(lp))
    if rc:
        raise OracleError("colour plan")
    return rv[:nr.value].copy(), lr[:nl].copy(), lp[:nl].copy()


def write_colorized_ply(path, X, colors, centers):
    """orc_write_colorized_ply: X (n, 3) in landmark id order, colors (n, 3) uint8 or None, centers (m, 3) in pose-id
    order."""
    X = np.ascontiguousarray(X, np.float64).reshape(-1, 3)
    cen = np.ascontiguousarray(centers, np.float64).reshape(-1, 3)
    col = None if colors is None else np.ascontiguousarray(colors, np.uint8).reshape(-1, 3)
    rc = lib().orc_write_colorized_ply(len(X), _p(X), None if col is None else _p(col), len(cen), _p(cen), path.encode())
    if rc:
        raise OracleError("PLY writer")


def undistort_image(model, focal, ppx, ppy, disto, rgb):
    """orc_undistort_image of one H x W x 3 uint8 image; disto padded with zeros to 5."""
    rgb = np.ascontiguousarray(rgb, np.uint8)
    h, w = rgb.shape[:2]
    d = np.zeros(5)
    d[:len(disto)] = disto
    out = np.empty_like(rgb)
    rc = lib().orc_undistort_image(int(model), float(focal), float(ppx), float(ppy), _p(d), _p(rgb), w, h, _p(out))
    if rc:
        raise OracleError("undistortion")
    return out
