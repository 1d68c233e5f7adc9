"""-m gpu: r3d_sfm_structure_from_tracks and r3d_sfm_remove_outliers on every camera model, through the C ABI and
SfmData, against the independent float64 / long-double reference in structure_ref.py.  Scenes are seeded and built
with resection_scenes.distort / project only."""
import numpy as np
import pytest

import structure_ref as sr
from resection_scenes import DISTO, project

pytestmark = pytest.mark.gpu

FOCAL, W, H = 2200.0, 2000, 1500
R3D_ERR_UNSUPPORTED = -5


def _ppx(g):
    """Principal point of intrinsic group g; float32-exact, so an uploaded pixel can sit on it exactly."""
    return 1000.5 + 3.25 * g, 749.75 - 2.5 * g


def _cam(model, g, R, t):
    return (model, DISTO[model], FOCAL) + _ppx(g) + (R, t)


def _upload(gpu_ctx, xy_per_view):
    gpu_ctx.clear_regions()
    for v, xy in xy_per_view.items():
        gpu_ctx.upload_regions(v, np.zeros((max(len(xy), 1), 64), np.uint8), np.asarray(xy, np.float32).reshape(-1, 2))


def _tracks(r3dlib, tviews, tfeats):
    """Tracks whose k-th member is the chain tviews[k][0] - tviews[k][1] - ... (features tfeats[k]), as pairwise matches."""
    I, J, fi, fj = [], [], [], []
    for vs, fs in zip(tviews, tfeats):
        o = np.argsort(vs)
        vs, fs = np.asarray(vs)[o], np.asarray(fs)[o]
        I.append(vs[:-1]); J.append(vs[1:]); fi.append(fs[:-1]); fj.append(fs[1:])
    I, J, fi, fj = (np.concatenate(a).astype(np.int64) for a in (I, J, fi, fj))
    o = np.lexsort((fj, fi, J, I))
    I, J, fi, fj = I[o], J[o], fi[o], fj[o]
    key = I * 100000 + J
    first = np.r_[0, np.nonzero(np.diff(key))[0] + 1]
    pairs = np.stack([I[first], J[first]], 1)
    ofs = np.r_[first, len(I)].astype(np.uint64)
    m = np.zeros(len(I), r3dlib.indmatch_dtype)
    m["i"], m["j"] = fi, fj
    return r3dlib.Tracks.build(r3dlib.Matches.from_csr(pairs, ofs, m), 2)


def _f32_error(xy32):
    """Per-coordinate error (normalised units) of float32-rounded pixels, with room for the undistortion's gain."""
    return 1.5 * 0.5 * np.spacing(np.abs(np.asarray(xy32, np.float32))).max(1).astype(np.float64) / FOCAL


def _check_points(cams, ofs, cam, xy, X_gpu, X_ref, X_true):
    """X_gpu within 1e-9 rel. (plus the K1 / K3 bisection's bound) of the reference, and within the float32 pixel
    budget of the truth."""
    sigma = sr.sensitivity(cams, ofs, cam, X_ref)
    bis = np.zeros(len(cam))
    for c in np.unique(cam):
        m = cam == c
        model, disto, f, ppx, ppy = cams[c][:5]
        bis[m] = sr.bisection_error(model, disto, f, ppx, ppy, xy[m])
    tol = 1e-9 * np.linalg.norm(X_ref, axis=1) + sr.point_bound(ofs, bis, sigma)
    err = np.linalg.norm(X_gpu - X_ref, axis=1)
    bad = np.nonzero(err > tol)[0]
    assert len(bad) == 0, "%d points off the reference, worst rel. %.3g" % (len(bad), (err / np.linalg.norm(X_ref, axis=1)).max())
    budget = tol + sr.point_bound(ofs, _f32_error(xy), sigma)
    err_t = np.linalg.norm(X_gpu - X_true, axis=1)
    assert (err_t <= budget).all(), "max truth error %.3g vs budget %.3g" % (err_t.max(), budget[np.argmax(err_t - budget)])


def _landmark_table(lms, owner):
    """{reference landmark index: (X, [(view, feat)])} of SfmData landmarks; owner[(view, feat)] -> reference index."""
    out = {}
    for lm in lms:
        v, f = lm["obs"][0][:2]
        out[owner[(v, f)]] = (np.array(lm["X"]), sorted((o[0], o[1]) for o in lm["obs"]))
    return out


# ---- 1. every model, one intrinsic group, noise-free --------------------------------------------------------------------
@pytest.mark.parametrize("model", [1, 2, 3, 4, 5])
def test_structure_from_tracks_per_model(gpu_ctx, r3dlib, model):
    rng = np.random.default_rng(700 + model)
    n_cams, M = 4, 2000
    sd = r3dlib.SfmData()
    d = list(DISTO[model])
    sd.add_intrinsic(0, model, W, H, FOCAL, *_ppx(0), disto=d)
    cams = []
    for v, C in enumerate(sr.sphere_centres(rng, n_cams, 8.0)):
        R, t = sr.look_at(C, rng.normal(size=3) * 0.2)
        cams.append(_cam(model, 0, R, t))
        sd.add_view(v, "image%06d.jpg" % v, W, H, id_intrinsic=0, id_pose=v)
        sd.add_pose(v, R, C)
    X = rng.uniform(-2.0, 2.0, (M, 3))
    xy = {v: project(model, FOCAL, *_ppx(0), DISTO[model], cams[v][5], cams[v][6], X).astype(np.float32) for v in range(n_cams)}
    _upload(gpu_ctx, xy)
    tracks = _tracks(r3dlib, [list(range(n_cams))] * M, [[l] * n_cams for l in range(M)])
    assert gpu_ctx.structure_from_tracks(sd, tracks) == 0
    got = _landmark_table(sd.landmarks(), {(v, l): l for v in range(n_cams) for l in range(M)})
    assert sorted(got) == list(range(M))
    ofs = np.arange(M + 1) * n_cams
    cam = np.tile(np.arange(n_cams), M)
    obs = np.stack([xy[v][l] for l in range(M) for v in range(n_cams)]).astype(np.float64)
    Xr, okr = sr.triangulate(cams, ofs, cam, sr.undistort_pixels(cams, cam, obs))
    assert okr.all()
    _check_points(cams, ofs, cam, obs, np.stack([got[l][0] for l in range(M)]), Xr, X)


# ---- 2. mixed models, long tracks, edge cases, more than 100 000 landmarks -------------------------------------------
# Most landmarks of this scene are rejected (points behind a camera): a kept landmark is read back through
# r3d_sfm_get_landmark, which walks the structure map from its start, so reading all of them costs O(kept^2).
MODELS = (4, 5, 3)                    # intrinsic group g: Brown T2, fisheye, radial K3
N_REG = 200                           # regular views 0 .. 199, pose v, intrinsic v % 3
V_NOPOSE, V_NOINTR, V_SHARED = 200, 201, 202
AB = ((203, 204), (205, 206))         # camera pairs A, B looking along +z, B 5 units ahead of A


def _mixed_scene(seed=11, n_random=15_000, n_ab=85_003):
    rng = np.random.default_rng(seed)
    views = {}                       # view -> (camera index | None, intrinsic id, pose id)
    cams = []
    for v, C in enumerate(sr.sphere_centres(rng, N_REG, 8.0, spread=0.9)):
        R, t = sr.look_at(C, rng.normal(size=3) * 0.2)
        cams.append(_cam(MODELS[v % 3], v % 3, R, t))
        views[v] = (v, v % 3, v)
    views[V_NOPOSE] = (None, 0, 9999)                # pose id that is never defined
    views[V_NOINTR] = (None, 77, 201)                # intrinsic id that is never defined (its pose is)
    views[V_SHARED] = (5, 5 % 3, 5)                  # shares view 5's pose and intrinsic
    for p, (va, vb) in enumerate(AB):                # a point between A and B is in front of A and behind B
        for v, dz, g in ((va, 0.0, 0), (vb, 5.0, 1 + p)):
            cams.append(_cam(MODELS[g], g, np.eye(3), -np.array([50.0 + 10.0 * p, 0.0, dz])))
            views[v] = (len(cams) - 1, g, v)
    cam_of = {v: c for v, (c, _, _) in views.items()}
    # tracks: (views, true point, pixel overrides {view: pixel})
    L, named = [], {}
    lens = np.where(rng.uniform(size=n_random) < 0.97, rng.integers(2, 7, n_random), rng.integers(7, 41, n_random))
    lens[rng.choice(n_random, 24, replace=False)] = rng.integers(100, N_REG + 1, 24)
    lens[:2] = N_REG, 2
    Xr = rng.uniform(-1.5, 1.5, (n_random, 3))
    for k in range(n_random):
        L.append((rng.choice(N_REG, lens[k], replace=False), Xr[k], {}))
    for v in range(6):                               # a pixel exactly on the principal point of each group (twice)
        C = -cams[v][5].T @ cams[v][6]
        X = C + cams[v][5][2] * rng.uniform(6.0, 10.0)
        others = [u for u in rng.choice(N_REG, 4, replace=False) if u != v][:2]
        L.append((np.r_[v, others], X, {v: _ppx(v % 3)}))
    special = rng.uniform(-1.5, 1.5, (6, 3))
    for name, vs in (("nopose_1", [V_NOPOSE, 10]), ("nopose_2", [V_NOPOSE, 10, 11]), ("nointr_1", [V_NOINTR, 12]),
                     ("nointr_2", [V_NOINTR, 12, 13, V_NOPOSE]), ("shared_3", [5, V_SHARED, 20]),
                     ("shared_5", [5, V_SHARED, 20, 21, 22])):
        named[name] = len(L)
        L.append((np.array(vs), special[len(named) - 1], {}))
    # A - B tracks: 95 % between the two cameras (rejected), the rest in front of both
    z = np.where(rng.uniform(size=n_ab) < 0.95, rng.uniform(0.8, 4.2, n_ab), rng.uniform(6.0, 12.0, n_ab))
    lat = 0.15 * np.minimum(z, np.abs(5.0 - z))[:, None] * rng.uniform(-1, 1, (n_ab, 2))
    pair = rng.integers(0, len(AB), n_ab)
    named["ab_first"] = len(L)
    for k in range(n_ab):
        L.append((np.array(AB[pair[k]]), np.array([50.0 + 10.0 * pair[k] + lat[k, 0], lat[k, 1], z[k]]), {}))
    # feature ids (an observation's rank in its view) and pixels per view; views without a camera get view 0's pixels
    n = np.array([len(t[0]) for t in L])
    first = np.r_[0, np.cumsum(n)]
    all_v = np.concatenate([t[0] for t in L])
    all_X = np.repeat(np.stack([t[1] for t in L]), n, axis=0)
    feat = np.empty(len(all_v), np.int64)
    pix = np.empty((len(all_v), 2))
    for v in views:
        m = all_v == v
        feat[m] = np.arange(m.sum())
        model, disto, f, ppx, ppy, R, t = cams[cam_of[v] if cam_of[v] is not None else 0]
        pix[m] = project(model, f, ppx, ppy, disto, R, t, all_X[m])
    for k, (vs, _, over) in enumerate(L):
        for v, p in over.items():
            pix[first[k] + list(vs).index(v)] = p
    tf = [feat[first[k]:first[k + 1]] for k in range(len(L))]
    xy = {v: pix[all_v == v].astype(np.float32) for v in views}
    return rng, views, cams, cam_of, L, tf, xy, named


def _mixed_sfm(r3dlib, views, cams, shared_intr=None):
    sd = r3dlib.SfmData()
    for g, model in enumerate(MODELS):
        sd.add_intrinsic(g, model, W, H, FOCAL, *_ppx(g), disto=list(DISTO[model]))
    for v, (c, gi, pid) in views.items():
        sd.add_view(v, "image%06d.jpg" % v, W, H, id_intrinsic=(shared_intr if v == V_SHARED and shared_intr is not None else gi),
                    id_pose=pid)
        if c is not None and pid == v:
            sd.add_pose(v, cams[c][5], -cams[c][5].T @ cams[c][6])
    sd.add_pose(V_NOINTR, np.eye(3), np.zeros(3))
    return sd


def test_structure_from_tracks_mixed_models(gpu_ctx, r3dlib):
    rng, views, cams, cam_of, L, tf, xy, named = _mixed_scene()
    n_lm = len(L)
    assert n_lm > 100_000 and n_lm % 128 != 0 and max(len(t[0]) for t in L) == N_REG
    _upload(gpu_ctx, xy)
    tracks = _tracks(r3dlib, [t[0] for t in L], tf)
    assert len(tracks) == n_lm
    sd = _mixed_sfm(r3dlib, views, cams)
    rejected = gpu_ctx.structure_from_tracks(sd, tracks)
    owner = {(int(v), int(f)): k for k, (t, fs) in enumerate(zip(L, tf)) for v, f in zip(t[0], fs)}
    got = _landmark_table(sd.landmarks(), owner)
    # reference: the observations of views with a pose and an intrinsic, in track order
    ofs, cam, obs, Xt = [0], [], [], []
    for k, (vs, X, _) in enumerate(L):
        for v, f in zip(vs, tf[k]):
            if v not in (V_NOPOSE, V_NOINTR):
                cam.append(cam_of[v]); obs.append(xy[v][f])
        ofs.append(len(cam)); Xt.append(X)
    ofs, cam, obs, Xt = np.array(ofs), np.array(cam), np.array(obs, np.float64), np.array(Xt)
    Xr, okr = sr.triangulate(cams, ofs, cam, sr.undistort_pixels(cams, cam, obs))
    assert sorted(got) == np.nonzero(okr)[0].tolist()
    assert rejected == int((~okr).sum())
    assert not okr[named["nopose_1"]] and not okr[named["nointr_1"]]
    ab = okr[named["ab_first"]:]
    assert 0.9 * len(ab) < (~ab).sum() < len(ab) and okr[:named["ab_first"]].sum() == named["ab_first"] - 2
    # a kept landmark keeps all its observations, also those of views that could not take part
    for k in (named["nopose_2"], named["nointr_2"], named["shared_3"], named["shared_5"]):
        assert k in got and got[k][1] == sorted((int(v), int(f)) for v, f in zip(L[k][0], tf[k]))
    kept = np.nonzero(okr)[0]
    sel = np.concatenate([np.arange(ofs[k], ofs[k + 1]) for k in kept])
    ofs_k = np.r_[0, np.cumsum(np.diff(ofs)[kept])]
    _check_points(cams, ofs_k, cam[sel], obs[sel], np.stack([got[k][0] for k in kept]), Xr[kept], Xt[kept])


def test_pose_shared_by_two_intrinsics_is_unsupported(gpu_ctx, r3dlib):
    rng, views, cams, cam_of, L, tf, xy, _ = _mixed_scene(n_random=200, n_ab=100)
    _upload(gpu_ctx, xy)
    tracks = _tracks(r3dlib, [t[0] for t in L], tf)
    sd = _mixed_sfm(r3dlib, views, cams, shared_intr=(5 + 1) % 3)   # view 202: pose of view 5, another intrinsic
    with pytest.raises(r3dlib.R3DError) as e:
        gpu_ctx.structure_from_tracks(sd, tracks)
    assert e.value.code == R3D_ERR_UNSUPPORTED


# ---- 3. outlier filters on landmarks set directly ------------------------------------------------------------------------
N_OV, N_TWIN = 30, 10                 # regular views 0 .. 29; view 30 + k sits about 1 degree from view k


def _outlier_scene(seed=23, n_random=3000, thr=4.0):
    rng = np.random.default_rng(seed)
    cams = []
    centres = sr.sphere_centres(rng, N_OV, 8.0, spread=0.9)
    for k in range(N_TWIN):
        C = centres[k]
        side = np.cross(C, rng.normal(size=3))
        centres = np.r_[centres, [C + side / np.linalg.norm(side) * 8.0 * np.radians(1.0)]]
    for v, C in enumerate(centres):
        R, t = sr.look_at(C)
        cams.append(_cam(MODELS[v % 3], v % 3, R, t))
    lms = []                                          # (views, X, pixels)

    def pixels(vs, X, kinds):
        out = []
        for v, kind in zip(vs, kinds):
            model, disto, f, ppx, ppy, R, t = cams[v]
            p = project(model, f, ppx, ppy, disto, R, t, X[None])[0]
            a = rng.uniform(0, 2 * np.pi)
            mag = {"clean": abs(rng.normal()) * 0.3, "gross": rng.uniform(30, 300),
                   "near": thr + rng.choice([-1, 1]) * rng.uniform(0.3, 3.0)}[kind]
            out.append(p + mag * np.array([np.cos(a), np.sin(a)]))
        return out

    for _ in range(n_random):
        vs = rng.choice(N_OV, rng.integers(2, 9), replace=False)
        kinds = rng.choice(["clean", "gross", "near"], len(vs), p=[0.7, 0.08, 0.22])
        X = rng.uniform(-1.5, 1.5, 3)
        lms.append((vs, X, pixels(vs, X, kinds)))
    for k in range(N_TWIN):
        X = rng.uniform(-1.0, 1.0, 3)
        far = (k + 15) % N_OV
        for vs, kinds in (([k, N_OV + k], ["clean"] * 2),                   # angle ~1 deg: removed
                          ([k, N_OV + k, far], ["clean", "clean", "gross"]),  # passes only with the dropped observation
                          ([k, N_OV + k, far], ["clean"] * 3),              # kept
                          ([k, far, (far + 1) % N_OV], ["gross", "gross", "clean"])):  # too short after pruning
            vs = np.array(vs)
            lms.append((vs, X, pixels(vs, X, kinds)))
    return cams, lms


@pytest.mark.parametrize("min_track_length,min_angle_deg", [(2, 2.0), (3, 2.0), (2, 0.0)])
def test_remove_outliers_mixed_models(gpu_ctx, r3dlib, min_track_length, min_angle_deg):
    thr = 4.0
    cams, lms = _outlier_scene(thr=thr)
    sd = r3dlib.SfmData()
    for g, model in enumerate(MODELS):
        sd.add_intrinsic(g, model, W, H, FOCAL, *_ppx(g), disto=list(DISTO[model]))
    for v, c in enumerate(cams):
        sd.add_view(v, "image%06d.jpg" % v, W, H, id_intrinsic=v % 3, id_pose=v)
        sd.add_pose(v, c[5], -c[5].T @ c[6])
    for l, (vs, X, px) in enumerate(lms):
        sd.add_landmark(l, X, [(int(v), l, float(p[0]), float(p[1])) for v, p in zip(vs, px)])
    rm_obs, rm_lm = gpu_ctx.remove_outliers(sd, thr, min_track_length, min_angle_deg)
    ofs = np.r_[0, np.cumsum([len(t[0]) for t in lms])]
    cam = np.concatenate([t[0] for t in lms])
    xy = np.concatenate([t[2] for t in lms])
    X = np.stack([t[1] for t in lms])
    ref = sr.remove_outliers(cams, ofs, cam, xy, X, thr, min_track_length, min_angle_deg)
    amb = ref["ambiguous"]
    got = {lm["id"]: sorted((o[0], o[1]) for o in lm["obs"]) for lm in sd.landmarks()}
    assert set(got) - amb == set(ref["keep"]) - amb
    for l, kept in ref["keep"].items():
        if l not in amb:
            assert got[l] == sorted((int(cam[o]), l) for o in kept), l
    assert abs(rm_obs - ref["rm_obs"]) <= len(amb) and abs(rm_lm - ref["rm_lm"]) <= len(amb)
    if not amb:
        assert (rm_obs, rm_lm) == (ref["rm_obs"], ref["rm_lm"])
    # the scene exercises every branch: drops by residual, by length, by angle in either pass
    assert ref["rm_obs"] > 500 and len(ref["keep"]) > 1000
    first = len(lms) - 4 * N_TWIN                   # the hand-built landmarks, four per twin pair
    twin_only, second_pass = [first + 4 * k for k in range(N_TWIN)], [first + 4 * k + 1 for k in range(N_TWIN)]
    assert all(first + 4 * k + 3 not in got for k in range(N_TWIN))
    if min_angle_deg > 0:
        assert not any(l in got for l in twin_only + second_pass)
    elif min_track_length == 2:
        assert all(l in got for l in twin_only + second_pass)
