"""ctypes wrapper of the CPU ORACLE of the rotation-averaging step (oracle/_build/liboracle_rotavg.so, oracle/rotavg.mk).

TEST INFRASTRUCTURE ONLY, like pyoracle: importable from tests/, __graft_entry__.smoke() and scripts/bench_rotavg.py.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.pyoracle import BAOptions, _p, default_ba_options
from oracle.pyoracle_relpose import RELPOSE_NO_MODEL, RELPOSE_OK, relpose_dtype  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liboracle_rotavg.so")


def build(force=False):
    """Compile liboracle_rotavg.so (and liboracle_relpose.so / liboracle.so, which it links) with oracle/rotavg.mk."""
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "rotavg.mk"] + (["-B"] if force else []))
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_rotavg_cycle_error.restype = C.c_float
        _lib.orc_rotavg_triplets.restype = C.c_int64
        _lib.orc_rotavg_l2_subspace.restype = C.c_uint32
    return _lib


class RotavgOptions(C.Structure):
    _fields_ = [("method", C.c_int), ("max_angular_error_deg", C.c_double), ("refine", C.c_int), ("lm", BAOptions)]


class RotavgSummary(C.Structure):
    _fields_ = [("success", C.c_int), ("n_edges", C.c_uint64), ("n_triplets", C.c_uint64), ("n_valid_triplets", C.c_uint64),
                ("n_kept_edges", C.c_uint64), ("n_kept_views", C.c_uint32), ("init_iterations", C.c_uint32),
                ("lm_iterations", C.c_uint32), ("lm_successful_steps", C.c_uint32), ("lm_termination", C.c_int),
                ("lm_initial_cost", C.c_double), ("lm_final_cost", C.c_double), ("ms_triplets", C.c_double),
                ("ms_init", C.c_double), ("ms_refine", C.c_double), ("ms_device_total", C.c_double), ("ms_host", C.c_double)]


class OracleError(RuntimeError):
    def __init__(self, code):
        super().__init__("oracle rotation averaging returned %d" % code)
        self.code = code


def rotation_averaging(rel, n_views, refine=True, max_angular_error_deg=5.0, method=0, n_threads=0, **lm):
    """orc_rotation_averaging: (rotations (n_views,3,3), view_kept, edge_kept, edge_support, summary dict); raises
    OracleError(-1 invalid / -5 unsupported)."""
    rel = np.ascontiguousarray(rel, relpose_dtype)
    o = RotavgOptions()
    o.method = method
    o.max_angular_error_deg = max_angular_error_deg
    o.refine = int(refine)
    o.lm = default_ba_options(huber_a=0.0, refine_intrinsics=0, n_threads=1)
    for k, v in lm.items():
        setattr(o.lm, k, v)
    rot = np.zeros((max(n_views, 1), 3, 3))
    vk = np.zeros(max(n_views, 1), np.uint8)
    ek = np.zeros(max(len(rel), 1), np.uint8)
    sup = np.zeros(max(len(rel), 1), np.uint32)
    s = RotavgSummary()
    rc = lib().orc_rotation_averaging(_p(rel), C.c_uint64(len(rel)), C.c_uint32(n_views), C.byref(o), _p(rot), _p(vk), _p(ek),
                                      _p(sup), C.byref(s), C.c_int(n_threads))
    if rc:
        raise OracleError(rc)
    summ = {k: getattr(s, k) for k, _ in RotavgSummary._fields_}
    return rot[:n_views], vk[:n_views].astype(bool), ek[:len(rel)].astype(bool), sup[:len(rel)].copy(), summ


def cycle_error(Rij, Rjk, Rik):
    """The triplet error (float degrees) of the cycle R_ik^T R_jk R_ij, as both implementations compute it."""
    a, b, c = [np.ascontiguousarray(x, np.float64) for x in (Rij, Rjk, Rik)]
    return float(lib().orc_rotavg_cycle_error(_p(a), _p(b), _p(c)))


def triplets(ij, R, n_views, thr=5.0, cap=None):
    """Every triangle {i < j < k}: (tri (T,3) view ids, err (T,) float32, valid (T,) bool).  R[e] = R_ij of (min, max)."""
    ij = np.ascontiguousarray(ij, np.uint32).reshape(-1, 2)
    R = np.ascontiguousarray(R, np.float64).reshape(-1, 9)
    cap = len(ij) ** 2 if cap is None else cap
    tri = np.zeros((max(cap, 1), 3), np.uint32)
    err = np.zeros(max(cap, 1), np.float32)
    val = np.zeros(max(cap, 1), np.uint8)
    n = lib().orc_rotavg_triplets(_p(ij), _p(R), C.c_uint64(len(ij)), C.c_uint32(n_views), C.c_float(thr), _p(tri), _p(err), _p(val),
                                  C.c_uint64(cap))
    assert n <= cap
    return tri[:n].copy(), err[:n].copy(), val[:n].astype(bool)


def largest_biedge_component(ij, n_views):
    """Boolean mask of the views in the largest 2-edge-connected component of the graph ij (E x 2)."""
    ij = np.ascontiguousarray(ij, np.uint32).reshape(-1, 2)
    kept = np.zeros(max(n_views, 1), np.uint8)
    lib().orc_largest_biedge_component(_p(ij), C.c_uint64(len(ij)), C.c_uint32(n_views), _p(kept))
    return kept[:n_views].astype(bool)


def l2_subspace(ab, R, m, n_threads=0):
    """The linear step on local ids: (M (3m,3m), Q (3m,3) orthonormal basis of its 3 smallest eigenvectors, iterations)."""
    ab = np.ascontiguousarray(ab, np.uint32).reshape(-1, 2)
    R = np.ascontiguousarray(R, np.float64).reshape(-1, 9)
    M = np.zeros((3 * m, 3 * m))
    Q = np.zeros((3 * m, 3))
    it = lib().orc_rotavg_l2_subspace(_p(ab), _p(R), C.c_uint64(len(ab)), C.c_uint32(m), _p(M), _p(Q), C.c_int(n_threads))
    return M, Q, int(it)
