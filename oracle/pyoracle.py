"""ctypes wrapper of the CPU ORACLE (oracle/_build/liboracle.so).

TEST INFRASTRUCTURE ONLY -- importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package (regard3d_b200) never imports this.
PARITY UNPINNED: see oracle/oracle.h.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "liboracle.so")


_REF_LIOP_PATH = os.path.join(_HERE, "_ref", "libvlliop_ref.so")
REFERENCE_ROOT = os.environ.get("R3D_REFERENCE", "/root/reference")


def build(force=False):
    """Compile the oracle with the committed Makefile (g++ -O3 -fopenmp -ffp-contract=off; make tracks the sources)
    and, when the reference tree is present (the build container; never on the GPU box), oracle/_ref."""
    subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    build_ref()
    return _LIB_PATH


def build_ref():
    """oracle/_ref/libvlliop_ref.so: the reference's own vendored LIOP (src/thirdparty/liop/vl_liop.c) compiled from
    the source where it lies.  Returns the path, or None when neither the reference tree nor a prebuilt file exists."""
    if os.path.exists(os.path.join(REFERENCE_ROOT, "src", "thirdparty", "liop", "vl_liop.c")):
        subprocess.check_call(["make", "-C", _HERE, "-s", "ref", "REFERENCE=" + REFERENCE_ROOT])
    return _REF_LIOP_PATH if os.path.exists(_REF_LIOP_PATH) else None


_lib = None


class IndMatch(C.Structure):
    _fields_ = [("i", C.c_uint32), ("j", C.c_uint32)]


indmatch_dtype = np.dtype([("i", np.uint32), ("j", np.uint32)])


class BAProblem(C.Structure):
    _fields_ = [
        ("n_cams", C.c_uint32), ("n_pts", C.c_uint32), ("n_intr", C.c_uint32),
        ("n_obs", C.c_uint64),
        ("poses", C.c_void_p), ("intrinsics", C.c_void_p), ("points", C.c_void_p),
        ("obs_cam", C.c_void_p), ("obs_pt", C.c_void_p), ("cam_intr", C.c_void_p),
        ("obs_xy", C.c_void_p),
        ("intr_model", C.c_void_p), ("intrinsics_ext", C.c_void_p), ("n_priors", C.c_uint32),
        ("prior_cam", C.c_void_p), ("prior_center", C.c_void_p), ("prior_weight", C.c_void_p),
    ]


class BAOptions(C.Structure):
    _fields_ = [
        ("max_iterations", C.c_uint32), ("huber_a", C.c_double), ("refine_intrinsics", C.c_int),
        ("function_tolerance", C.c_double), ("gradient_tolerance", C.c_double),
        ("parameter_tolerance", C.c_double), ("initial_radius", C.c_double), ("n_threads", C.c_int),
        ("prior_huber_a", C.c_double),
    ]


class BASummary(C.Structure):
    _fields_ = [
        ("iterations", C.c_uint32), ("successful_steps", C.c_uint32),
        ("initial_cost", C.c_double), ("final_cost", C.c_double), ("termination", C.c_int),
        ("seconds_total", C.c_double), ("seconds_linear", C.c_double),
    ]


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_l2_f32.restype = C.c_float
        _lib.orc_l2_u8.restype = C.c_float
        _lib.orc_match_distance_ratio.restype = C.c_int64
        _lib.orc_match_pairs.restype = C.c_int64
        _lib.orc_coord_dedup.restype = C.c_int64
        _lib.orc_acransac_F.restype = C.c_int64
        _lib.orc_filter_pairs_F.restype = C.c_int64
        _lib.orc_filter_pairs_H.restype = C.c_int64
        _lib.orc_acransac_H.restype = C.c_int64
        _lib.orc_acransac_E.restype = C.c_int64
        _lib.orc_filter_pairs_E.restype = C.c_int64
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _dt(desc):
    if desc.dtype == np.float32:
        return 0
    if desc.dtype == np.uint8:
        return 1
    raise TypeError("descriptors must be float32 or uint8")


def l2(a, b):
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b)
    if a.dtype == np.uint8:
        return float(lib().orc_l2_u8(_p(a), _p(b), C.c_uint64(a.size)))
    a = a.astype(np.float32, copy=False)
    b = b.astype(np.float32, copy=False)
    return float(lib().orc_l2_f32(_p(a), _p(b), C.c_uint64(a.size)))


def search_neighbours(db, q, n_threads=0):
    """ArrayMatcherBruteForce::SearchNeighbours(NN=2): returns (idx[nq,2] int32, dist[nq,2] f32) or None."""
    db = np.ascontiguousarray(db)
    q = np.ascontiguousarray(q)
    nq = q.shape[0]
    idx = np.zeros((nq, 2), np.int32)
    dist = np.zeros((nq, 2), np.float32)
    rc = lib().orc_search_neighbours(_p(db), C.c_uint32(db.shape[0]), _p(q), C.c_uint32(nq),
                                     C.c_uint32(db.shape[1]), _dt(db), _p(idx), _p(dist),
                                     C.c_int(n_threads))
    return None if rc else (idx, dist)


def match_distance_ratio(descI, xyI, descJ, xyJ, ratio, n_threads=0):
    descI = np.ascontiguousarray(descI)
    descJ = np.ascontiguousarray(descJ)
    xyI = np.ascontiguousarray(xyI, np.float32)
    xyJ = np.ascontiguousarray(xyJ, np.float32)
    out = np.zeros(max(1, descJ.shape[0]), indmatch_dtype)
    n = lib().orc_match_distance_ratio(_p(descI), _p(xyI), C.c_uint32(descI.shape[0]), _p(descJ),
                                       _p(xyJ), C.c_uint32(descJ.shape[0]),
                                       C.c_uint32(descI.shape[1] if descI.ndim == 2 else 0),
                                       _dt(descI), C.c_float(ratio), _p(out), C.c_int(n_threads))
    return out[:n].copy()


def _ptr_array(arrs):
    T = C.c_void_p * len(arrs)
    return T(*[a.ctypes.data for a in arrs])


def match_pairs(descs, xys, pairs, ratio, n_threads=0):
    """Matcher_Regions::Match twin.  Returns (pair_ofs[P+1] uint64, matches structured array)."""
    descs = [np.ascontiguousarray(d) for d in descs]
    xys = [np.ascontiguousarray(x, np.float32) for x in xys]
    pairs = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
    P = pairs.shape[0]
    ns = np.array([d.shape[0] for d in descs], np.uint32)
    dim = max([d.shape[1] for d in descs if d.ndim == 2 and d.shape[0] > 0] + [0])
    cap = int(sum(int(ns[j]) for _, j in pairs)) + 1
    out = np.zeros(cap, indmatch_dtype)
    ofs = np.zeros(P + 1, np.uint64)
    dt = _dt(descs[0])
    n = lib().orc_match_pairs(_ptr_array(descs), _ptr_array(xys), _p(ns), C.c_uint32(len(descs)),
                              C.c_uint32(dim), dt, _p(pairs), C.c_uint64(P), C.c_float(ratio),
                              _p(ofs), _p(out), C.c_uint64(cap), C.c_int(n_threads))
    if n < 0:
        raise RuntimeError("orc_match_pairs overflow")
    return ofs, out[:n].copy()


def cascade_match_pairs(descs, xys, pairs, ratio, n_threads=0):
    """Cascade_Hashing_Matcher_Regions::Match twin (oracle_cascade.cpp); same return shape as match_pairs."""
    descs = [np.ascontiguousarray(d) for d in descs]
    xys = [np.ascontiguousarray(x, np.float32) for x in xys]
    pairs = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
    P = pairs.shape[0]
    ns = np.array([d.shape[0] for d in descs], np.uint32)
    dim = max([d.shape[1] for d in descs if d.ndim == 2 and d.shape[0] > 0] + [0])
    cap = int(sum(int(ns[j]) for _, j in pairs)) + 1
    out = np.zeros(cap, indmatch_dtype)
    ofs = np.zeros(P + 1, np.uint64)
    fn = lib().orc_cascade_match_pairs
    fn.restype = C.c_int64
    n = fn(_ptr_array(descs), _ptr_array(xys), _p(ns), C.c_uint32(len(descs)), C.c_uint32(dim), _dt(descs[0]),
           _p(pairs), C.c_uint64(P), C.c_float(ratio), _p(ofs), _p(out), C.c_uint64(cap), C.c_int(n_threads))
    if n < 0:
        raise RuntimeError("orc_cascade_match_pairs overflow")
    return ofs, out[:n].copy()


def cascade_projections(dim):
    out = np.zeros((dim + 60, dim), np.float32)
    lib().orc_cascade_projections(C.c_uint32(dim), _p(out))
    return out


def coord_dedup(m, xyI, xyJ):
    m = np.ascontiguousarray(m, indmatch_dtype).copy()
    xyI = np.ascontiguousarray(xyI, np.float32)
    xyJ = np.ascontiguousarray(xyJ, np.float32)
    n = lib().orc_coord_dedup(_p(m), C.c_int64(m.shape[0]), _p(xyI), _p(xyJ))
    return m[:n].copy()


def seven_point(x1, x2):
    x1 = np.ascontiguousarray(x1, np.float64)
    x2 = np.ascontiguousarray(x2, np.float64)
    F = np.zeros((3, 3, 3), np.float64)
    n = lib().orc_seven_point(_p(x1), _p(x2), _p(F))
    return F[:n].copy()


def acransac_F(xI, xJ, wI, hI, wJ, hJ, precision_px=4.0, max_iter=2048):
    xI = np.ascontiguousarray(xI, np.float64)
    xJ = np.ascontiguousarray(xJ, np.float64)
    M = xI.shape[0]
    inl = np.zeros(max(M, 1), np.uint32)
    F = np.zeros((3, 3), np.float64)
    info = np.zeros(3, np.float64)
    n = lib().orc_acransac_F(_p(xI), _p(xJ), C.c_uint32(M), C.c_uint32(wI), C.c_uint32(hI),
                             C.c_uint32(wJ), C.c_uint32(hJ), C.c_double(precision_px),
                             C.c_uint32(max_iter), _p(inl), _p(F), _p(info))
    return inl[:n].copy(), F, info


def filter_pairs_F(xys, widths, heights, pairs, put_ofs, put, precision_px=4.0, max_iter=2048,
                   n_threads=0, model="F"):
    xys = [np.ascontiguousarray(x, np.float32) for x in xys]
    pairs = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
    P = pairs.shape[0]
    widths = np.ascontiguousarray(widths, np.uint32)
    heights = np.ascontiguousarray(heights, np.uint32)
    put_ofs = np.ascontiguousarray(put_ofs, np.uint64)
    put = np.ascontiguousarray(put, indmatch_dtype)
    out = np.zeros(max(1, put.shape[0]), indmatch_dtype)
    out_ofs = np.zeros(P + 1, np.uint64)
    fn = lib().orc_filter_pairs_F if model == "F" else lib().orc_filter_pairs_H
    n = fn(_ptr_array(xys), _p(widths), _p(heights), C.c_uint32(len(xys)),
                                 _p(pairs), C.c_uint64(P), _p(put_ofs), _p(put),
                                 C.c_double(precision_px), C.c_uint32(max_iter), _p(out_ofs), _p(out),
                                 C.c_int(n_threads))
    return out_ofs, out[:n].copy()


def filter_pairs_H(xys, widths, heights, pairs, put_ofs, put, precision_px=4.0, max_iter=2048, n_threads=0):
    return filter_pairs_F(xys, widths, heights, pairs, put_ofs, put, precision_px, max_iter, n_threads, model="H")


def filter_pairs_E(xys, widths, heights, Ks, pairs, put_ofs, put, precision_px=4.0, max_iter=2048, n_threads=0):
    """Ks: n_views x 3 (f, ppx, ppy); f <= 0 = no valid pinhole intrinsic."""
    xys = [np.ascontiguousarray(x, np.float32) for x in xys]
    pairs = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
    P = pairs.shape[0]
    widths = np.ascontiguousarray(widths, np.uint32)
    heights = np.ascontiguousarray(heights, np.uint32)
    Ks = np.ascontiguousarray(Ks, np.float64)
    put_ofs = np.ascontiguousarray(put_ofs, np.uint64)
    put = np.ascontiguousarray(put, indmatch_dtype)
    out = np.zeros(max(1, put.shape[0]), indmatch_dtype)
    out_ofs = np.zeros(P + 1, np.uint64)
    n = lib().orc_filter_pairs_E(_ptr_array(xys), _p(widths), _p(heights), _p(Ks), C.c_uint32(len(xys)),
                                 _p(pairs), C.c_uint64(P), _p(put_ofs), _p(put),
                                 C.c_double(precision_px), C.c_uint32(max_iter), _p(out_ofs), _p(out),
                                 C.c_int(n_threads))
    return out_ofs, out[:n].copy()


def acransac_E(xI, xJ, wI, hI, wJ, hJ, Kpair, precision_px=4.0, max_iter=2048):
    """Kpair = (f1, ppx1, ppy1, f2, ppx2, ppy2).  Returns inliers, F (= K2^-T E K1^-1), info."""
    xI = np.ascontiguousarray(xI, np.float64)
    xJ = np.ascontiguousarray(xJ, np.float64)
    Kpair = np.ascontiguousarray(Kpair, np.float64)
    M = xI.shape[0]
    inl = np.zeros(max(M, 1), np.uint32)
    F = np.zeros((3, 3), np.float64)
    info = np.zeros(3, np.float64)
    n = lib().orc_acransac_E(_p(xI), _p(xJ), C.c_uint32(M), C.c_uint32(wI), C.c_uint32(hI),
                             C.c_uint32(wJ), C.c_uint32(hJ), _p(Kpair), C.c_double(precision_px),
                             C.c_uint32(max_iter), _p(inl), _p(F), _p(info))
    return inl[:n].copy(), F, info


def five_point(b1, b2):
    """Bearing vectors (5x3 each) -> list of 3x3 essential matrices (b2^T E b1 = 0)."""
    b1 = np.ascontiguousarray(b1, np.float64)
    b2 = np.ascontiguousarray(b2, np.float64)
    E = np.zeros((10, 3, 3), np.float64)
    n = lib().orc_five_point(_p(b1), _p(b2), _p(E))
    return [E[k].copy() for k in range(n)]


def four_point(x1, x2):
    x1 = np.ascontiguousarray(x1, np.float64)
    x2 = np.ascontiguousarray(x2, np.float64)
    H = np.zeros((3, 3), np.float64)
    n = lib().orc_four_point(_p(x1), _p(x2), _p(H))
    return H if n else None


def acransac_H(xI, xJ, wI, hI, wJ, hJ, precision_px=4.0, max_iter=2048):
    xI = np.ascontiguousarray(xI, np.float64)
    xJ = np.ascontiguousarray(xJ, np.float64)
    M = xI.shape[0]
    inl = np.zeros(max(M, 1), np.uint32)
    H = np.zeros((3, 3), np.float64)
    info = np.zeros(3, np.float64)
    n = lib().orc_acransac_H(_p(xI), _p(xJ), C.c_uint32(M), C.c_uint32(wI), C.c_uint32(hI),
                             C.c_uint32(wJ), C.c_uint32(hJ), C.c_double(precision_px),
                             C.c_uint32(max_iter), _p(inl), _p(H), _p(info))
    return inl[:n].copy(), H, info


def save_feat(path, xyso):
    xyso = np.ascontiguousarray(xyso, np.float32)
    return lib().orc_save_feat(path.encode(), _p(xyso), C.c_uint32(xyso.shape[0]))


def load_feat(path, cap=1 << 22):
    buf = np.zeros((cap, 4), np.float32)
    n = C.c_uint32(0)
    rc = lib().orc_load_feat(path.encode(), _p(buf), C.c_uint32(cap), C.byref(n))
    if rc:
        raise IOError(path)
    return buf[: n.value].copy()


def save_desc(path, d):
    d = np.ascontiguousarray(d, np.float32)
    return lib().orc_save_desc_f32(path.encode(), _p(d), C.c_uint64(d.shape[0]), C.c_uint32(d.shape[1]))


def load_desc(path, dim, cap=1 << 22):
    buf = np.zeros((cap, dim), np.float32)
    n = C.c_uint64(0)
    rc = lib().orc_load_desc_f32(path.encode(), _p(buf), C.c_uint64(cap), C.c_uint32(dim), C.byref(n))
    if rc:
        raise IOError(path)
    return buf[: n.value].copy()


def save_matches_txt(path, pairs, pair_ofs, m):
    pairs = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
    pair_ofs = np.ascontiguousarray(pair_ofs, np.uint64)
    m = np.ascontiguousarray(m, indmatch_dtype)
    return lib().orc_save_matches_txt(path.encode(), _p(pairs), C.c_uint64(pairs.shape[0]),
                                      _p(pair_ofs), _p(m))


def _ba_struct(p):
    s = BAProblem()
    s.n_cams = p["poses"].shape[0]
    s.n_pts = p["points"].shape[0]
    s.n_intr = p["intrinsics"].shape[0]
    s.n_obs = p["obs_xy"].shape[0]
    for k in ("poses", "intrinsics", "points", "obs_cam", "obs_pt", "cam_intr", "obs_xy"):
        setattr(s, k, p[k].ctypes.data)
    ba_optional_fields(s, p)
    return s


def ba_optional_fields(s, p):
    """intr_model / intrinsics_ext / priors of a BA problem dict (all optional) -> the C struct."""
    if p.get("intr_model") is not None:
        p["intr_model"] = np.ascontiguousarray(p["intr_model"], np.uint8)
        s.intr_model = p["intr_model"].ctypes.data
    if p.get("intrinsics_ext") is not None:
        p["intrinsics_ext"] = np.ascontiguousarray(p["intrinsics_ext"], np.float64)
        s.intrinsics_ext = p["intrinsics_ext"].ctypes.data
    if p.get("prior_cam") is not None and len(p["prior_cam"]):
        p["prior_cam"] = np.ascontiguousarray(p["prior_cam"], np.uint32)
        p["prior_center"] = np.ascontiguousarray(p["prior_center"], np.float64)
        p["prior_weight"] = np.ascontiguousarray(p["prior_weight"], np.float64)
        s.n_priors = len(p["prior_cam"])
        s.prior_cam = p["prior_cam"].ctypes.data
        s.prior_center = p["prior_center"].ctypes.data
        s.prior_weight = p["prior_weight"].ctypes.data


def ba_prepare(poses, intrinsics, points, obs_cam, obs_pt, cam_intr, obs_xy):
    return {
        "poses": np.ascontiguousarray(poses, np.float64).copy(),
        "intrinsics": np.ascontiguousarray(intrinsics, np.float64).copy(),
        "points": np.ascontiguousarray(points, np.float64).copy(),
        "obs_cam": np.ascontiguousarray(obs_cam, np.uint32),
        "obs_pt": np.ascontiguousarray(obs_pt, np.uint32),
        "cam_intr": np.ascontiguousarray(cam_intr, np.uint32),
        "obs_xy": np.ascontiguousarray(obs_xy, np.float64),
    }


def default_ba_options(max_iterations=500, huber_a=16.0, refine_intrinsics=1, n_threads=0, prior_huber_a=0.0):
    o = BAOptions()
    o.max_iterations = max_iterations
    o.huber_a = huber_a
    o.refine_intrinsics = refine_intrinsics
    o.function_tolerance = 1e-6
    o.gradient_tolerance = 1e-10
    o.parameter_tolerance = 1e-8
    o.initial_radius = 1e4
    o.n_threads = n_threads
    o.prior_huber_a = prior_huber_a
    return o


def bundle_adjust(p, opts=None):
    """In-place on the dict from ba_prepare().  Returns (summary dict, cost_trace)."""
    opts = opts or default_ba_options()
    s = _ba_struct(p)
    summ = BASummary()
    trace = np.full(opts.max_iterations + 1, np.nan, np.float64)
    rc = lib().orc_bundle_adjust(C.byref(s), C.byref(opts), C.byref(summ), _p(trace))
    if rc:
        raise RuntimeError("orc_bundle_adjust rc=%d" % rc)
    d = {k: getattr(summ, k) for k, _ in BASummary._fields_}
    return d, trace[: summ.iterations + 1].copy()


def ba_residuals(p):
    s = _ba_struct(p)
    res = np.zeros((p["obs_xy"].shape[0], 2), np.float64)
    lib().orc_ba_residuals(C.byref(s), _p(res))
    return res


def ba_jacobian_model(model, intr, ext, pose, X, obs):
    intr, pose, X, obs = [np.ascontiguousarray(a, np.float64) for a in (intr, pose, X, obs)]
    ext = None if ext is None else np.ascontiguousarray(ext, np.float64)
    r = np.zeros(2)
    J = np.zeros((2, 15))
    lib().orc_ba_jacobian_model(C.c_int(model), _p(intr), None if ext is None else _p(ext), _p(pose), _p(X), _p(obs), _p(r), _p(J))
    return r, J


def ba_prior(pose, center, weight):
    pose, center, weight = [np.ascontiguousarray(a, np.float64) for a in (pose, center, weight)]
    r = np.zeros(3)
    J = np.zeros((3, 6))
    lib().orc_ba_prior(_p(pose), _p(center), _p(weight), _p(r), _p(J))
    return r, J


def ba_jacobian(intr, pose, X, obs):
    intr, pose, X, obs = [np.ascontiguousarray(a, np.float64) for a in (intr, pose, X, obs)]
    r = np.zeros(2)
    J = np.zeros((2, 15))
    lib().orc_ba_jacobian(_p(intr), _p(pose), _p(X), _p(obs), _p(r), _p(J))
    return r, J


def num_threads():
    return lib().orc_num_threads()


# ---- LIOP-144 descriptor stage (SURVEY.md 8f-1) --------------------------------------------------------------
LIOP_SIDE = 41


def liop_process(patch):
    """Restatement of r3d_vl_liopdesc_process on one 41x41 float32 patch -> desc[144]."""
    patch = np.ascontiguousarray(patch, np.float32).reshape(LIOP_SIDE * LIOP_SIDE)
    desc = np.zeros(144, np.float32)
    lib().orc_liop_process(_p(patch), _p(desc))
    return desc


_ref_liop = None


def liop_ref_available():
    return build_ref() is not None


def liop_ref_process(patches):
    """THE REFERENCE ITSELF: r3d_vl_liopdesc_new_basic(41) + r3d_vl_liopdesc_process of oracle/_ref (compiled from
    /root/reference/src/thirdparty/liop/vl_liop.c) on n patches -> (n, 144)."""
    global _ref_liop
    if _ref_liop is None:
        path = build_ref()
        if path is None:
            raise RuntimeError("oracle/_ref/libvlliop_ref.so is not built and the reference tree is absent")
        L = C.CDLL(path)
        L.r3d_vl_liopdesc_new_basic.restype = C.c_void_p
        L.r3d_vl_liopdesc_new_basic.argtypes = [C.c_size_t]
        L.r3d_vl_liopdesc_process.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.r3d_vl_liopdesc_delete.argtypes = [C.c_void_p]
        L.r3d_vl_liopdesc_get_dimension.restype = C.c_size_t
        L.r3d_vl_liopdesc_get_dimension.argtypes = [C.c_void_p]
        _ref_liop = L
    L = _ref_liop
    patches = np.ascontiguousarray(patches, np.float32).reshape(-1, LIOP_SIDE * LIOP_SIDE)
    h = L.r3d_vl_liopdesc_new_basic(LIOP_SIDE)
    assert L.r3d_vl_liopdesc_get_dimension(h) == 144
    out = np.zeros((len(patches), 144), np.float32)
    for k in range(len(patches)):
        L.r3d_vl_liopdesc_process(h, out[k].ctypes.data, patches[k].ctypes.data)
    L.r3d_vl_liopdesc_delete(h)
    return out


def liop_affine(x, y, size, angle, factor):
    M = np.zeros(6, np.float32)
    lib().orc_liop_affine(C.c_float(x), C.c_float(y), C.c_float(size), C.c_float(angle), C.c_float(factor), _p(M))
    return M.reshape(2, 3)


def liop_warp(img, M):
    img = np.ascontiguousarray(img, np.float32)
    M = np.ascontiguousarray(M, np.float32).reshape(6)
    out = np.zeros((LIOP_SIDE, LIOP_SIDE), np.float32)
    lib().orc_liop_warp(_p(img), C.c_int(img.shape[1]), C.c_int(img.shape[0]), _p(M), _p(out))
    return out


def liop_blur(patch):
    patch = np.ascontiguousarray(patch, np.float32).reshape(LIOP_SIDE, LIOP_SIDE)
    out = np.zeros((LIOP_SIDE, LIOP_SIDE), np.float32)
    lib().orc_liop_blur(_p(patch), _p(out))
    return out


def liop_describe(img, kps, factor, want_patches=False):
    """extractLIOPFeatures twin: kps (n, 4) = x, y, size (diameter), angle (degrees) -> (n, 144) [, (n, 41, 41)]."""
    img = np.ascontiguousarray(img, np.float32)
    kps = np.ascontiguousarray(kps, np.float32).reshape(-1, 4)
    n = len(kps)
    desc = np.zeros((n, 144), np.float32)
    patches = np.zeros((n, LIOP_SIDE, LIOP_SIDE), np.float32) if want_patches else None
    lib().orc_liop_describe(_p(img), C.c_int(img.shape[1]), C.c_int(img.shape[0]), _p(kps), C.c_uint64(n), C.c_float(factor),
                            _p(desc), _p(patches) if want_patches else None)
    return (desc, patches) if want_patches else desc


# ---- steps either side of BA (SURVEY.md 8f-3) ----------------------------------------------------------------------
def tracks_build(pairs, pair_ofs, m, min_length=2):
    """TracksBuilder Build + Filter + ExportToSTL -> {track id: {view: feature}}."""
    pairs = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
    pair_ofs = np.ascontiguousarray(pair_ofs, np.uint64)
    m = np.ascontiguousarray(m, indmatch_dtype)
    cap_n = 2 * len(m) + 1
    ids = np.zeros(cap_n, np.uint32)
    ofs = np.zeros(cap_n + 1, np.uint64)
    views = np.zeros(cap_n, np.uint32)
    feats = np.zeros(cap_n, np.uint32)
    lib().orc_tracks_build.restype = C.c_int64
    T = lib().orc_tracks_build(_p(pairs), C.c_uint64(len(pairs)), _p(pair_ofs), _p(m), C.c_uint32(min_length), _p(ids), _p(ofs),
                               _p(views), _p(feats), C.c_uint64(cap_n), C.c_uint64(cap_n))
    assert T >= 0
    return {int(ids[k]): dict(zip(views[int(ofs[k]):int(ofs[k + 1])].tolist(), feats[int(ofs[k]):int(ofs[k + 1])].tolist()))
            for k in range(T)}


def _ext(intr_ext, n_intr):
    """intrinsics_ext per intrinsic group (t1 t2 for Brown, k4 0 for the fisheye); None: zeros."""
    return None if intr_ext is None else np.ascontiguousarray(np.asarray(intr_ext, np.float64).reshape(n_intr, 2))


def triangulate_landmarks(obs_ofs, obs_cam, obs_xy, poses, cam_intr, intrinsics, intr_model=None, intr_ext=None):
    obs_ofs = np.ascontiguousarray(obs_ofs, np.uint64)
    obs_cam = np.ascontiguousarray(obs_cam, np.uint32)
    obs_xy = np.ascontiguousarray(obs_xy, np.float64)
    poses = np.ascontiguousarray(poses, np.float64)
    cam_intr = np.ascontiguousarray(cam_intr, np.uint32)
    intrinsics = np.ascontiguousarray(intrinsics, np.float64)
    n = len(obs_ofs) - 1
    X = np.zeros((n, 3))
    ok = np.zeros(n, np.uint8)
    im = None if intr_model is None else np.ascontiguousarray(intr_model, np.uint8)
    ext = _ext(intr_ext, len(intrinsics))
    lib().orc_triangulate_landmarks(C.c_uint32(n), _p(obs_ofs), _p(obs_cam), _p(obs_xy), _p(poses), _p(cam_intr), _p(intrinsics),
                                    None if im is None else _p(im), None if ext is None else _p(ext), _p(X), _p(ok))
    return X, ok.astype(bool)


def landmark_checks(obs_ofs, obs_cam, obs_xy, poses, cam_intr, intrinsics, X, thr_px, intr_model=None, intr_ext=None):
    obs_ofs = np.ascontiguousarray(obs_ofs, np.uint64)
    obs_cam = np.ascontiguousarray(obs_cam, np.uint32)
    obs_xy = np.ascontiguousarray(obs_xy, np.float64)
    poses = np.ascontiguousarray(poses, np.float64)
    cam_intr = np.ascontiguousarray(cam_intr, np.uint32)
    intrinsics = np.ascontiguousarray(intrinsics, np.float64)
    X = np.ascontiguousarray(X, np.float64)
    n = len(obs_ofs) - 1
    keep = np.zeros(len(obs_cam), np.uint8)
    ang = np.zeros(n)
    im = None if intr_model is None else np.ascontiguousarray(intr_model, np.uint8)
    ext = _ext(intr_ext, len(intrinsics))
    lib().orc_landmark_checks(C.c_uint32(n), _p(obs_ofs), _p(obs_cam), _p(obs_xy), _p(poses), _p(cam_intr), _p(intrinsics),
                              None if im is None else _p(im), None if ext is None else _p(ext), _p(X), C.c_double(thr_px),
                              _p(keep), _p(ang))
    return keep.astype(bool), ang
