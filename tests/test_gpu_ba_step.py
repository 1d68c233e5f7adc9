"""One bundle-adjustment LM step (r3d_debug_ba_step: the code r3d_bundle_adjust runs per iteration) against the float64
reference of ba_step_ref.py: the scaled gradient and diag(J^T J) of k_ba_eval / k_ba_apply_scale, the reduced camera
system S and its right-hand side after both Schur kernels, the prior U blocks and k_ba_finish_S, every point's V^-1,
the step of the Cholesky solve and k_ba_backsub, and the norms and model cost change of k_ba_update.

The library sums with fp64 atomics, so no result is bit-reproducible and a fixed tolerance would be either loose or
flaky.  Each value is held to |gpu - ref| <= c u A instead, where A is the same sum over absolute values (ba_step_ref.py)
and c a small multiple of the number of terms.  The step is held to its backward error on the full, unreduced system,
which does not depend on the conditioning of S."""
import numpy as np
import pytest

import ba_step_ref as ref
from regard3d_b200 import synth

U = ref.U
W, H, F = 1920, 1080, 1.1 * 1920


def _arrays(prob):
    out = {}
    for k, v in prob.items():
        if k == "truth" or v is None:
            continue
        dt = np.uint32 if k in ("obs_cam", "obs_pt", "cam_intr", "prior_cam") else np.uint8 if k == "intr_model" else np.float64
        out[k] = np.ascontiguousarray(np.array(v), dt)
    return out


def _ring(n_cams, tracks, seed, n_intr=1, cam_intr=None):
    """Cameras on synth's ring around the scene; point k is observed by the cameras in tracks[k], in that order (a
    repeated camera sees the point twice; an empty track leaves the point without observations).  Initial state:
    truth + noise, as synth.make_ba_problem."""
    rng = np.random.default_rng(seed)
    poses, Rs, ts = synth.ring_cameras(n_cams, rng)
    X = rng.uniform([3.5, 3.5, 1.0], [6.5, 6.5, 3.0], (len(tracks), 3))
    oc, op, oxy = [], [], []
    for k, cams in enumerate(tracks):
        for c in cams:
            pc = Rs[c] @ X[k] + ts[c]
            oc.append(c)
            op.append(k)
            oxy.append(F * pc[:2] / pc[2] + [W / 2, H / 2] + 0.5 * rng.standard_normal(2))
    intr = np.tile([F, W / 2, H / 2, 0.0, 0.0, 0.0], (n_intr, 1))
    intr[:, 0] *= 1 + 0.01 * rng.standard_normal(n_intr)
    return {"poses": poses + 1e-2 * rng.standard_normal(poses.shape), "intrinsics": intr,
            "points": X + 5e-2 * rng.standard_normal(X.shape), "obs_cam": np.array(oc, np.uint32),
            "obs_pt": np.array(op, np.uint32), "obs_xy": np.array(oxy).reshape(-1, 2),
            "cam_intr": np.zeros(n_cams, np.uint32) if cam_intr is None else np.asarray(cam_intr, np.uint32)}


def _groups(prob, n, factor=0.005):
    prob["intrinsics"] = np.repeat(prob["intrinsics"], n, 0).copy()
    prob["intrinsics"][:, 0] *= 1 + factor * np.arange(n)
    prob["cam_intr"] = (np.arange(len(prob["poses"])) % n).astype(np.uint32)
    return prob


def _models(model, n_pts=500):
    # the problem of test_gpu_ba.py::test_ba_other_camera_models_equal_oracle
    prob = synth.make_ba_problem(n_cams=10, n_pts=n_pts, obs_per_pt=4, seed=40 + model, outlier_frac=0.01)
    prob["intrinsics"] = np.repeat(prob["intrinsics"], 2, 0).copy()
    prob["cam_intr"] = (np.arange(10) % 2).astype(np.uint32)
    prob["intr_model"] = np.array([model, 3], np.uint8)
    prob["intrinsics_ext"] = np.array([[1e-4, -2e-4], [0.0, 0.0]])
    return prob


def _dup_three_groups():
    # the problem of test_gpu_ba.py::test_ba_camera_sees_point_twice_and_three_groups
    prob = _groups(synth.make_ba_problem(n_cams=9, n_pts=300, obs_per_pt=4, seed=23, outlier_frac=0.0), 3)
    dup = np.arange(0, 80, 4)
    prob["obs_cam"] = np.concatenate([prob["obs_cam"], prob["obs_cam"][dup]]).astype(np.uint32)
    prob["obs_pt"] = np.concatenate([prob["obs_pt"], prob["obs_pt"][dup]]).astype(np.uint32)
    prob["obs_xy"] = np.concatenate([prob["obs_xy"], prob["obs_xy"][dup] + 0.3])
    return prob


def _tracks():
    """Track lengths 1, 2, 4, 32 (the batched kernel's maximum), 33 and 200 on a ring of 200 cameras; a camera that
    sees a 4-track point twice."""
    rng = np.random.default_rng(61)
    tracks = []
    for L, n in ((1, 6), (2, 20), (4, 300), (32, 6), (33, 4), (200, 3)):
        for _ in range(n):
            c0 = int(rng.integers(200))
            tracks.append([(c0 + 3 * j) % 200 for j in range(L)])
    tracks[30] = tracks[30] + [tracks[30][1]]
    return _ring(200, tracks, seed=62)


def _priors():
    """Pose-centre priors, one with a gross error and one on a camera (12) no observation reaches."""
    prob = synth.make_ba_problem(n_cams=13, n_pts=600, obs_per_pt=4, seed=51, outlier_frac=0.0)
    keep = prob["obs_cam"] != 12
    for k in ("obs_cam", "obs_pt", "obs_xy"):
        prob[k] = prob[k][keep]
    truth = prob["truth"]
    rng = np.random.default_rng(5)
    Cs = np.stack([-synth._rodrigues(truth["poses"][c, :3]).T @ truth["poses"][c, 3:] for c in range(13)])
    cams = np.array([0, 2, 3, 7, 11, 12], np.uint32)
    prob["prior_cam"] = cams
    prob["prior_center"] = Cs[cams] + 0.05 * rng.standard_normal((6, 3))
    prob["prior_center"][1] += 3.0
    prob["prior_weight"] = np.tile([1.0, 1.0, 2.0], (6, 1))
    return prob


def _orphans():
    """14 cameras and 2 intrinsic groups (nB = 96 = 3 * 32): camera 13 and group 1 unused, 5 points unobserved."""
    rng = np.random.default_rng(71)
    tracks = [sorted(rng.choice(13, int(rng.integers(2, 6)), replace=False).tolist()) for _ in range(200)]
    for k in (0, 57, 58, 120, 199):
        tracks[k] = []
    return _ring(14, tracks, seed=72, n_intr=2)


def _long_track_200():
    from test_gpu_ba import _long_track_problem
    return _long_track_problem(200, 3000, 12, 21)


# name -> (problem builder, options, expected (n_batches, n_long) of the default plan or None)
CASES = {
    "one_group": (lambda: synth.make_ba_problem(n_cams=8, n_pts=300, obs_per_pt=4, seed=3, outlier_frac=0.02), {}, None),
    "one_group_fixed_intrinsics": (lambda: synth.make_ba_problem(n_cams=8, n_pts=300, obs_per_pt=4, seed=3, outlier_frac=0.02),
                                   {"refine": 0}, None),
    "two_groups_alternating": (lambda: _groups(synth.make_ba_problem(n_cams=10, n_pts=500, obs_per_pt=4, seed=13), 2), {}, (None, 0)),
    "three_groups_and_duplicates": (_dup_three_groups, {}, None),
    "tracks_1_2_32_33_200": (_tracks, {}, (None, 8)),
    # 48 two-view points: 24 points per batch
    "batch_cut_by_points": (lambda: _ring(4, [[0, 1]] * 48, seed=81), {}, (2, 0)),
    # 8 points seen by all 32 cameras: 33 entries each (one group), 4 per batch
    "batch_cut_by_entries": (lambda: _ring(32, [list(range(32))] * 8, seed=82), {}, (2, 0)),
    # 6 points seen by 6 disjoint sets of 8 cameras: 9 new blocks per point (8 cameras and, once, the group), 4 per batch
    "batch_cut_by_blocks": (lambda: _ring(48, [list(range(8 * k, 8 * k + 8)) for k in range(6)], seed=83), {}, (2, 0)),
    "pinhole": (lambda: _models(1), {}, None),
    "radial_k1": (lambda: _models(2), {}, None),
    "radial_k3": (lambda: _models(3), {}, None),
    "brown_t2": (lambda: _models(4), {}, None),
    "fisheye": (lambda: _models(5), {}, None),  # test_gpu_ba.py's 2e-3 problem at its initial parameters
    "huber_outliers": (lambda: synth.make_ba_problem(n_cams=8, n_pts=300, obs_per_pt=4, seed=9, outlier_frac=0.1), {}, None),
    "trivial_loss_outliers": (lambda: synth.make_ba_problem(n_cams=8, n_pts=300, obs_per_pt=4, seed=9, outlier_frac=0.1),
                              {"huber_a": 0.0}, None),
    "priors": (_priors, {}, None),
    "priors_robust": (_priors, {"prior_huber_a": 0.5}, None),
    "orphans": (_orphans, {}, (None, 0)),
    "long_track_200": (_long_track_200, {}, None),  # test_gpu_ba.py's 5e-5 problem at its initial parameters
}
RADII = (1e4, 1e-2)

_ref_cache = {}


def _case(name, radius, oracle):
    key = (name, radius)
    if key not in _ref_cache:
        build, opts, expect = CASES[name]
        p = _arrays(build())
        o = dict(huber_a=16.0, refine=1, prior_huber_a=0.0)
        o.update(opts)
        _ref_cache[key] = (p, o, expect, ref.step(oracle, p, radius, **o))
    return _ref_cache[key]


def _run(ctx, p, o, radius, route):
    return ctx.debug_ba_step(p, radius, huber_a=o["huber_a"], refine_intrinsics=o["refine"], prior_huber_a=o["prior_huber_a"],
                             route=route)


def _bar(p):
    """c = 16 (longest track + 16): a small multiple of the number of terms in the longest sum."""
    longest = np.bincount(p["obs_pt"]).max() if len(p["obs_pt"]) else 1
    return 16.0 * (longest + 16)


def _ratio(got, want, A):
    """max |got - want| / (u A); inf where got is not finite."""
    got = np.asarray(got, np.float64)
    if not np.all(np.isfinite(got)):
        return np.inf
    err = np.abs(got - np.asarray(want))
    return float((err / np.maximum(U * np.asarray(A), np.finfo(float).tiny)).max()) if err.size else 0.0


def _step_ratios(r, R, p, o):
    """Every output of one r3d_debug_ba_step against the reference, as multiples of u A (delta: backward error in u)."""
    assert r["nB"] == R["nB"]
    q = {k: _ratio(r[k], R[k], R["A_" + k]) for k in ("g", "diag", "Vinv", "S", "rhs")}
    rel_du = np.divide(R["A_diag"], R["diag"], out=np.zeros_like(R["diag"]), where=R["diag"] > 0)
    q["scale"] = _ratio(r["scale"], R["scale"], R["scale"] * (1 + rel_du))
    q["gmax"] = _ratio(r["gmax"], R["gmax"], (R["A_g"] / R["scale"]).max())
    # the step: backward error on the unreduced system (H + D^2) delta = -g, normwise (Frobenius norm of H)
    d = r["delta"]
    Hn = np.sqrt(R["H"].multiply(R["H"]).sum())
    q["delta"] = np.inf if not np.all(np.isfinite(d)) else \
        np.linalg.norm(R["H"] @ d + R["g"]) / (U * (Hn * np.linalg.norm(d) + np.linalg.norm(R["g"])))
    # k_ba_update on the library's own step
    D2, g = R["D2"], R["g"]
    q["mcc"] = _ratio(r["model_cost_change"], 0.5 * np.sum(d * (D2 * d - g)), 0.5 * np.sum(np.abs(d) * (D2 * np.abs(d) + R["A_g"])))
    dx = d * R["scale"]
    q["dx"] = _ratio(r["dx_norm2"], dx @ dx, dx @ dx)
    x = np.concatenate([p["poses"].ravel(), p["intrinsics"].ravel() if o["refine"] else [], p["points"].ravel()])
    q["x"] = _ratio(r["x_norm2"], x @ x, x @ x)
    return q


def _fmt(q):
    return " ".join("%s %.3g" % kv for kv in q.items())


@pytest.mark.gpu
@pytest.mark.parametrize("radius", RADII)
@pytest.mark.parametrize("name", list(CASES))
def test_ba_step_equals_float64_reference(gpu_ctx, oracle, name, radius):
    from regard3d_b200 import capi
    p, o, expect, R = _case(name, radius, oracle)
    c = _bar(p)
    a = _run(gpu_ctx, p, o, radius, capi.SCHUR_PLAN)
    b = _run(gpu_ctx, p, o, radius, capi.SCHUR_CTA)
    qa, qb = _step_ratios(a, R, p, o), _step_ratios(b, R, p, o)
    # both routes: the same reduced system to the same bar
    qab = {"S": _ratio(a["S"], b["S"], 2 * R["A_S"]), "rhs": _ratio(a["rhs"], b["rhs"], 2 * R["A_rhs"])}
    print("\n%s r=%g c=%g batches %d long %d\n  plan %s\n  cta  %s\n  plan vs cta %s" % (
        name, radius, c, a["n_batches"], a["n_long"], _fmt(qa), _fmt(qb), _fmt(qab)))
    bad = ["%s %s %.3g" % (route, k, v) for route, q in (("plan", qa), ("cta", qb), ("plan-vs-cta", qab)) for k, v in q.items()
           if not v <= (c * np.sqrt(R["nparam"]) if k == "delta" else c)]
    assert not bad, "over the bar (c = %g): %s" % (c, ", ".join(bad))
    for r in (a, b):
        assert np.array_equal(r["S"], r["S"].T) and not r["not_pd"]
    # the all-CTA route puts every observed point through k_ba_schur_cta
    assert b["n_batches"] == 0 and b["n_long"] == len(np.unique(p["obs_pt"]))
    if expect is not None:
        nb, nl = expect
        if nb is not None:
            assert a["n_batches"] == nb
        assert a["n_long"] == nl


def test_case_structures():
    """The cases exercise what their names say (no GPU needed)."""
    p = _arrays(_tracks())
    lengths = np.bincount(p["obs_pt"], minlength=len(p["points"]))
    assert {1, 2, 32, 33, 200} <= set(lengths.tolist())
    q = _arrays(_orphans())
    assert (np.bincount(q["obs_pt"], minlength=len(q["points"])) == 0).sum() == 5
    assert 13 not in q["obs_cam"] and 6 * (14 + 2) % 32 == 0
    d = _arrays(_dup_three_groups())
    assert len(set(zip(d["obs_cam"].tolist(), d["obs_pt"].tolist()))) < len(d["obs_cam"])
    pr = _arrays(_priors())
    assert 12 in pr["prior_cam"] and 12 not in pr["obs_cam"]
    s = _arrays(CASES["huber_outliers"][0]())
    assert len(s["obs_xy"]) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("radius", RADII)
def test_points_without_observations_get_V_equal_D2_and_a_zero_step(gpu_ctx, oracle, radius):
    """No Schur kernel visits a point without observations; its V is D^2 alone (as the oracle has it), so its V^-1 is
    diag(1 / D^2) and, with g_p = 0, its step is exactly 0 whatever the memory held before."""
    from regard3d_b200 import capi
    p, o, _, R = _case("orphans", radius, oracle)
    orphan = np.nonzero(np.bincount(p["obs_pt"], minlength=len(p["points"])) == 0)[0]
    nB = R["nB"]
    D2 = R["D2"][nB:].reshape(-1, 3)[orphan]
    for route in (capi.SCHUR_PLAN, capi.SCHUR_CTA):
        # leave NaN in the device pool first (NaN points make NaN V^-1 everywhere): a step that read a V^-1 it never
        # wrote would come out NaN
        q = dict(p, points=np.full_like(p["points"], np.nan))
        _run(gpu_ctx, q, o, radius, route)
        r = _run(gpu_ctx, p, o, radius, route)
        Vi = r["Vinv"][orphan]
        assert np.allclose(Vi[:, [0, 1, 2], [0, 1, 2]], 1.0 / D2, rtol=4 * U, atol=0)
        assert not Vi[:, [0, 0, 1, 1, 2, 2], [1, 2, 0, 2, 0, 1]].any()
        step = r["delta"][nB:].reshape(-1, 3)[orphan]
        assert np.all(step == 0.0)


def _small_with_everything():
    prob = synth.make_ba_problem(n_cams=4, n_pts=20, obs_per_pt=3, seed=5, outlier_frac=0.15)
    prob["intrinsics"][0, 3:] = [0.02, -0.01, 0.003]
    prob["prior_cam"] = np.array([0, 2], np.uint32)
    prob["prior_center"] = np.array([[1.0, 2.0, 3.0], [-4.0, 0.5, 1.0]])
    prob["prior_weight"] = np.array([[1.0, 1.0, 2.0], [0.5, 0.5, 0.5]])
    return _arrays(prob)


def test_reference_gradient_is_the_cost_derivative(oracle):
    """The reference's unscaled gradient J^T r (Huber-corrected, with priors) against central differences of the cost."""
    p = _small_with_everything()
    R = ref.step(oracle, p, 1e4, huber_a=16.0, refine=1, prior_huber_a=2.0)
    assert (np.abs(R["r"]) > 0).all() and R["gmax"] > 0
    gu = R["g"] / R["scale"]
    nc, ni = len(p["poses"]), len(p["intrinsics"])
    blocks = [("poses", 0), ("intrinsics", 6 * nc), ("points", 6 * nc + 6 * ni)]
    for key, base in blocks:
        for j in range(p[key].size):
            x0 = p[key].flat[j]
            h = 1e-6 * max(1.0, abs(x0))
            q = {k: v.copy() for k, v in p.items()}
            q[key].flat[j] = x0 + h
            cp = ref.cost(oracle, q, 16.0, 2.0)
            q[key].flat[j] = x0 - h
            cm = ref.cost(oracle, q, 16.0, 2.0)
            num = (cp - cm) / (2 * h)
            assert abs(num - gu[base + j]) <= 1e-6 * abs(gu).max() + 1e-5 * abs(num), (key, j, num, gu[base + j])


def test_reference_schur_solve_equals_the_dense_solve(oracle):
    """On a small case the reference's reduced system, solved and back-substituted, is the dense solve of
    (J^T J + D^2) delta = -g; and its magnitudes bound what they stand for."""
    p = _small_with_everything()
    for radius in RADII:
        R = ref.step(oracle, p, radius, huber_a=16.0, refine=1, prior_huber_a=2.0)
        Hd = R["H"].toarray()
        Js = R["J"].toarray() * R["scale"]
        assert np.allclose(Hd, Js.T @ Js + np.diag(R["D2"]), rtol=0, atol=1e-12 * np.abs(Hd).max())
        dense = np.linalg.solve(Hd, -R["g"])
        d = ref.solve_reduced(R)
        assert np.linalg.norm(d - dense) <= 1e-9 * np.linalg.norm(dense)
        for k in ("g", "S", "rhs", "Vinv", "diag"):
            assert (np.abs(R[k]) <= R["A_" + k] * (1 + 1e-12)).all(), k
