"""ctypes wrapper of the CPU ORACLE of the translation-averaging step (oracle/_build/liboracle_transavg.so,
oracle/transavg.mk).

TEST INFRASTRUCTURE ONLY, like pyoracle: importable from tests/, __graft_entry__.smoke() and scripts/bench_transavg.py.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.pyoracle import BAOptions, _p, default_ba_options
from oracle.pyoracle_relpose import RELPOSE_NO_MODEL, RELPOSE_OK, relpose_dtype  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liboracle_transavg.so")

TRANSAVG_L1, TRANSAVG_L2_CHORDAL, TRANSAVG_SOFTL1 = 1, 2, 3


def build(force=False):
    """Compile liboracle_transavg.so (and the oracle libraries it links) with oracle/transavg.mk."""
    subprocess.check_call(["make", "-C", _HERE, "-s", "-f", "transavg.mk"] + (["-B"] if force else []))
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_softl1_rho.restype = C.c_double
        _lib.orc_softl1_rho.argtypes = [C.c_double, C.c_double, C.c_void_p]
        _lib.orc_transavg_edge.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
    return _lib


class TransavgOptions(C.Structure):
    _fields_ = [("method", C.c_int), ("softl1_loss", C.c_double), ("lm", BAOptions)]


class TransavgSummary(C.Structure):
    _fields_ = [("success", C.c_int), ("n_edges", C.c_uint64), ("n_kept_edges", C.c_uint64), ("n_kept_views", C.c_uint32),
                ("lm_iterations", C.c_uint32), ("lm_successful_steps", C.c_uint32), ("lm_termination", C.c_int),
                ("lm_initial_cost", C.c_double), ("lm_final_cost", C.c_double), ("ms_solve", C.c_double),
                ("ms_device_total", C.c_double), ("ms_host", C.c_double)]


class OracleError(RuntimeError):
    def __init__(self, code):
        super().__init__("oracle translation averaging returned %d" % code)
        self.code = code


def translation_averaging(rel, rotations, rot_kept, n_views, method=TRANSAVG_L2_CHORDAL, edge_use=None, softl1_loss=0.01,
                          n_threads=0, **lm):
    """orc_translation_averaging: (centers (n_views,3), translations (n_views,3), view_kept, edge_kept, summary dict);
    raises OracleError(-1 invalid / -5 unsupported).  lm: orc_ba_options fields (max_iterations / function_tolerance 0:
    the method's)."""
    rel = np.ascontiguousarray(rel, relpose_dtype)
    rot = np.ascontiguousarray(np.asarray(rotations, np.float64).reshape(-1, 3, 3))
    rk = np.ascontiguousarray(np.asarray(rot_kept).astype(np.uint8).ravel())
    assert len(rot) >= n_views and len(rk) >= n_views
    use = None if edge_use is None else np.ascontiguousarray(np.asarray(edge_use).astype(np.uint8).ravel())
    o = TransavgOptions()
    o.method = method
    o.softl1_loss = softl1_loss
    o.lm = default_ba_options(max_iterations=0, huber_a=0.0, refine_intrinsics=0, n_threads=1)
    o.lm.function_tolerance = 0.0
    for k, v in lm.items():
        setattr(o.lm, k, v)
    cen = np.zeros((max(n_views, 1), 3))
    tra = np.zeros((max(n_views, 1), 3))
    vk = np.zeros(max(n_views, 1), np.uint8)
    ek = np.zeros(max(len(rel), 1), np.uint8)
    s = TransavgSummary()
    rc = lib().orc_translation_averaging(_p(rel), C.c_uint64(len(rel)), None if use is None else _p(use), _p(rot), _p(rk),
                                         C.c_uint32(n_views), C.byref(o), _p(cen), _p(tra), _p(vk), _p(ek), C.byref(s),
                                         C.c_int(n_threads))
    if rc:
        raise OracleError(rc)
    summ = {k: getattr(s, k) for k, _ in TransavgSummary._fields_}
    return cen[:n_views], tra[:n_views], vk[:n_views].astype(bool), ek[:len(rel)].astype(bool), summ


def edge(method, xi, xj, s, edata):
    """One edge's raw residual (3,) and Jacobian (3, 7: x_I, x_J, s) by the solver's jets."""
    xi, xj = np.ascontiguousarray(xi, np.float64), np.ascontiguousarray(xj, np.float64)
    e = np.zeros(6)
    e[:len(edata)] = edata
    r = np.zeros(3)
    J = np.zeros((3, 7))
    lib().orc_transavg_edge(method, _p(xi), _p(xj), float(s), _p(e), _p(r), _p(J))
    return r, J


def softl1_rho(sq, a):
    """ceres::SoftLOneLoss(a) at s = |r|^2: (rho, rho')."""
    r1 = np.zeros(1)
    r0 = lib().orc_softl1_rho(float(sq), float(a), _p(r1))
    return r0, float(r1[0])
