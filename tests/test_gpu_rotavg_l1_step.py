"""-m gpu: one step of r3d_rotation_averaging_l1 (r3d_debug_rotavg_l1_step: the members the solver runs) against the
problem-built reference of rotavg_l1_step_ref.py.

Newton steps of l1decode_pd run from the start point and from late states of the restatement's trajectory
(rotavg_l1_ref.l1_regression on the device's residuals), where sigma spans many decades, on scenes whose n = m - 1 free
views sit on and across the 32-row tiles of dense_cholesky (31, 32, 33, 64, 65), a 140-view complete graph (degree 139:
k_l1_system's 128-thread loop goes round twice) and the 300-view bench problem (44 850 edges: the 1024-thread reductions
loop, P = max(E, n) = E).  Records come as (I, J) and (J, I) alike (rotavg_scenes stores half of them reversed).  Each
value is held to |gpu - ref| <= c u A (c in rotavg_l1_step_ref.bars), the solves to their normwise backward error, the
direction to the unreduced Newton system, and the ratio test, trial steps, accept / backtrack, next tau and state bit
for bit.  Also: residuals within 1e-6 of pi against the known rotation vector, b = 0 exactly (signed permutations),
IRLS updates below sqrt(eps) (the Taylor branch of exp), chained steps = the solver bit for bit, the not positive
definite path, and invalid states."""
import itertools

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg
from scipy.spatial.transform import Rotation

import rotavg_l1_ref as ref
import rotavg_l1_step_ref as sr
from regard3d_b200 import capi
from rotavg_scenes import banded_ring, complete_edges, make_problem

pytestmark = pytest.mark.gpu
U = sr.U


def _complete(m, seed, thr=5.0, out=0.1):
    return lambda: (make_problem(m, complete_edges(m), noise_deg=0.5, outlier_frac=out, seed=seed)[0], m, thr)


def _banded(m, seed):
    return lambda: (make_problem(m, banded_ring(m, 4), noise_deg=0.5, outlier_frac=0.05, seed=seed)[0], m, 180.0)


SCENES = {
    "complete32": _complete(32, 61, 180.0, 0.2),   # n = 31: the right-hand side row inside the last 32-row tile
    "complete33": _complete(33, 62),               # n = 32: the right-hand side row in a tile of its own
    "complete34": _complete(34, 63, 180.0, 0.2),   # n = 33: across it
    "banded65": _banded(65, 64),                   # n = 64
    "banded66": _banded(66, 65),                   # n = 65
    "complete140": _complete(140, 66),             # degree 139 > 128
    "bench300": lambda: (make_problem(300, complete_edges(300), noise_deg=0.5, outlier_frac=0.1, seed=7,
                                      outlier_min_deg=0.0)[0], 300, 5.0),
}
_cache = {}


def _scene(ctx, name):
    """(rel, n, threshold, the start's kind-0 step, the restatement's trajectory on its residuals)."""
    if name not in _cache:
        rel, n, thr = SCENES[name]()
        D0 = ctx.debug_rotavg_l1_step(rel, n, max_angular_error_deg=thr)
        sc = sr.Scene.from_device(D0)
        tr = []
        ref.l1_regression(sc.ab, D0["b"].reshape(-1, 3), sc.m, trace=tr.append)
        _cache[name] = (rel, n, thr, D0, tr)
    return _cache[name]


def _state(t):
    cm = lambda v: np.asarray(v)[1:].T.ravel()
    return (cm(t["x"]), t["Ax"].ravel(), t["u"].ravel(), t["lam1"].ravel(), t["lam2"].ravel(), cm(t["Atv"])), t["tau"]


def _fmt(q):
    return " ".join("%s %.3g" % kv for kv in sorted(q.items()))


def _check_b(D, sc):
    b, A = sr.residuals(sc, D["rotations0"])
    q = {"b": sr._ratio(D["b"], b, A)}
    B = D["b"].reshape(-1, 3)
    ex = {"cost": np.array_equal(D["cost"], (np.abs(B[:, 0]) + np.abs(B[:, 1])) + np.abs(B[:, 2])),
          "bmax": D["bmax"] == np.abs(D["b"]).max()}
    return q, ex


@pytest.mark.parametrize("name", list(SCENES))
def test_pd_step_equals_reference(gpu_ctx, name):
    """Every output of one Newton iteration at the start point and at late states against the reference."""
    rel, n, thr, D0, tr = _scene(gpu_ctx, name)
    sc = sr.Scene.from_device(D0)
    _, _, _, _, ab, _, views = ref.kept_problem(rel, n, thr)
    assert np.array_equal(D0["ab"], ab) and np.array_equal(D0["view_ids"], views)
    # the host's spanning tree sums its 3-term products in order; numpy's matmul need not
    assert np.abs(D0["rotations0"] - ref.spanning_tree_start(ab, D0["Rk"], sc.m)).max() <= 1e-13
    bad, worst = [], {}
    k = len(tr)
    for which in [None] + sorted({k // 2, k - 3, k - 1}):
        if which is None:
            D, (st, tau) = D0, (D0["state0"], D0["tau0"])
            want = sr.start_state(sc, D0["b"])
            assert all(np.array_equal(a, c) for a, c in zip(st[:5], want[:5]))
            worst["start_Atv"] = sr._ratio(st[5], want[5], sc.absAt @ (np.abs(want[3]) + np.abs(want[4])))
            assert D0["tau0"] == sr.PD_MU * (2.0 * sc.nr) / D0["sdg0"]
        else:
            st, tau = _state(tr[which])
            D = gpu_ctx.debug_rotavg_l1_step(rel, n, state=st, tau=tau, max_angular_error_deg=thr)
            assert all(np.array_equal(a, c) for a, c in zip(D["state0"], st)) and D["tau0"] == tau
        assert not D["not_pd"]
        q, ex = sr.check_pd(D, sc, D["b"], st, tau)
        qb, exb = _check_b(D, sc)
        qr, exr = sr.check_rotations(D, sc, D["rotations0"], D["state"][0] if D["accepted"] else st[0])
        q.update(qb); q.update(qr); ex.update(exb); ex.update(exr)
        bad += ["%s@%s: %s" % (name, which, s) for s in sr.over_bar(q, ex, sc)]
        for kk, v in q.items():
            worst[kk] = max(worst.get(kk, 0.0), v)
        print("\n%s state %s (n %d, E %d, trials %d, sigma %.1e..%.1e): %s" % (
            name, which, sc.n, sc.E, len(D["trials"]), D["sigx"].min(), D["sigx"].max(), _fmt(q)))
    print("%s worst: %s" % (name, _fmt(worst)))
    assert not bad, bad


@pytest.mark.parametrize("name", ["complete32", "banded66", "complete140", "bench300"])
def test_irls_step_equals_reference(gpu_ctx, name):
    """One IRLS iteration at the spanning-tree start: weights, assembled systems, solve, update."""
    rel, n, thr, D0, _ = _scene(gpu_ctx, name)
    D = gpu_ctx.debug_rotavg_l1_step(rel, n, kind=1, max_angular_error_deg=thr)
    sc = sr.Scene.from_device(D)
    assert not D["not_pd"] and np.array_equal(D["b"], D0["b"])
    q, ex = sr.check_irls(D, sc, 5.0)
    qr, exr = sr.check_rotations(D, sc, D["rotations0"], D["dx"])
    q.update(qr); ex.update(exr)
    print("\n%s IRLS: %s" % (name, _fmt(q)))
    assert not sr.over_bar(q, ex, sc), sr.over_bar(q, ex, sc)


def _exact_scene(m, seed, angles):
    """Views at the truth, relative rotations exact products with an error rotation exp(w_e) on some edges: the
    residual of edge e at the truth is w_e.  Returns (rel, truth by view id, {edge: w})."""
    rng = np.random.default_rng(seed)
    Rs = Rotation.random(m, random_state=seed).as_matrix()
    I, J, R, known = [], [], [], {}
    for e, (i, j) in enumerate(complete_edges(m)):
        Rij = Rs[j] @ Rs[i].T
        if e < len(angles):
            ax = rng.standard_normal(3)
            w = ax / np.linalg.norm(ax) * angles[e]
            known[(i, j)] = w
            Rij = Rs[j] @ Rotation.from_rotvec(w).as_matrix() @ Rs[i].T
        if e % 2:
            I.append(j); J.append(i); R.append(Rij.T)
        else:
            I.append(i); J.append(j); R.append(Rij)
    return capi.relative_pose_records(I, J, np.array(R)), Rs, known


def test_residuals_near_pi_against_known_rotation_vectors(gpu_ctx):
    """Gross outliers whose residual is within 1e-6 (and 1e-3) of pi (the tr < 0 branch of the log and its sign flip):
    b at the truth is the known rotation vector within the reference's bar, which allows for the log map's
    conditioning there; the Newton step from there passes the reference too."""
    m = 12
    angles = [np.pi - 1e-6, np.pi - 1e-7, np.pi - 1e-3, np.pi - 3e-7, 1e-9]
    rel, Rs, known = _exact_scene(m, 71, angles)
    D = gpu_ctx.debug_rotavg_l1_step(rel, m, rotations=Rs, max_angular_error_deg=180.0)
    sc = sr.Scene.from_device(D)
    B = D["b"].reshape(-1, 3)
    c = sr.bars(sc)["b"]
    want = np.zeros_like(B)
    for e, (a, b) in enumerate(D["ab"]):
        w = known.get((D["view_ids"][a], D["view_ids"][b]))
        if w is not None:
            want[e] = w
    _, A = sr.residuals(sc, D["rotations0"])
    assert sr._ratio(B.ravel(), want.ravel(), A) <= c
    assert (np.linalg.norm(B, axis=1) > np.pi - 2e-6).sum() == 3
    q, ex = sr.check_pd(D, sc, D["b"], D["state0"], D["tau0"])
    q.update(_check_b(D, sc)[0])
    print("\nnear pi: %s" % _fmt(q))
    assert not sr.over_bar(q, ex, sc), sr.over_bar(q, ex, sc)


def test_zero_residuals_return_x_zero(gpu_ctx):
    """Relative rotations that are exact signed permutation matrices: the spanning-tree start leaves b exactly 0, the
    call returns x = 0 with no iteration, and the solver does the same."""
    perms = []
    for p in itertools.permutations(range(3)):
        for s in itertools.product((1.0, -1.0), repeat=3):
            P = np.zeros((3, 3))
            P[range(3), p] = s
            if np.linalg.det(P) > 0:
                perms.append(P)
    m = 10
    rng = np.random.default_rng(5)
    Rs = np.array([perms[i] for i in rng.integers(0, len(perms), m)])
    I, J, R = [], [], []
    for (i, j) in complete_edges(m):
        I.append(j); J.append(i); R.append(Rs[i] @ Rs[j].T)
    rel = capi.relative_pose_records(I, J, np.array(R))
    D = gpu_ctx.debug_rotavg_l1_step(rel, m)
    assert D["b_zero"] and not D["b"].any() and D["bmax"] == 0.0 and D["xmax"] == 0.0
    assert np.array_equal(D["rotations"], D["rotations0"]) and not D["trials"]
    _, _, _, _, S = gpu_ctx.rotation_averaging_l1(rel, m)
    assert S["pd_iterations"] == 0 and S["l1_iterations"] == 1 and S["termination"] == 0 and S["final_l1_cost"] == 0.0


def test_irls_update_below_sqrt_eps(gpu_ctx):
    """Rotations 1e-9 from the truth of a noise-free scene: the IRLS update is below sqrt(eps) (the Taylor branch of
    exp) and the rotated views match scipy's exp within the bar."""
    m = 12
    rel, Rs, _ = _exact_scene(m, 72, [])
    rng = np.random.default_rng(9)
    start = np.array([R @ Rotation.from_rotvec(rng.standard_normal(3) * 3e-10).as_matrix() for R in Rs])
    start = np.array([s @ Rs[0].T for s in start])
    start[0] = np.eye(3)
    D = gpu_ctx.debug_rotavg_l1_step(rel, m, kind=1, rotations=start)
    sc = sr.Scene.from_device(D)
    X = D["dx"].reshape(3, sc.n).T
    assert 0 < np.linalg.norm(X, axis=1).max() < np.sqrt(np.finfo(float).eps)
    q, ex = sr.check_irls(D, sc, 5.0)
    qr, exr = sr.check_rotations(D, sc, D["rotations0"], D["dx"])
    q.update(qr); ex.update(exr)
    print("\ntiny IRLS update (max |x| %.2g): %s" % (D["xmax"], _fmt(q)))
    assert not sr.over_bar(q, ex, sc), sr.over_bar(q, ex, sc)


def _chain(ctx, rel, n, opts):
    """rotation_averaging_l1 replayed by debug steps with the solver's stopping rules."""
    S = dict(l1_iterations=0, pd_iterations=0, pd_backtracks=0, irls_iterations=0, termination=1)
    R = None
    full = lambda D: _to_views(D, n)
    for _ in range(opts.get("l1_max_iterations", 32)):
        D = ctx.debug_rotavg_l1_step(rel, n, rotations=R, **opts)
        if not D["b_zero"]:
            assert not D["sdg0"] < sr.PD_TOL
            it = 0
            while True:
                it += 1
                S["pd_iterations"] += 1
                if D["not_pd"]:
                    S["termination"] = 2
                    return S, R
                S["pd_backtracks"] += len(D["trials"]) - (1 if D["accepted"] else 0)
                if not D["accepted"] or D["sdg"] < sr.PD_TOL or it >= sr.PD_MAX_ITER:
                    break
                D = ctx.debug_rotavg_l1_step(rel, n, rotations=R, state=D["state"], tau=D["tau"], **opts)
        R = full(D)
        S["l1_iterations"] += 1
        if D["xmax"] <= opts.get("tolerance", 1e-5):
            S["termination"] = 0
            break
    S["termination"] = 1
    for _ in range(opts.get("irls_max_iterations", 32)):
        D = ctx.debug_rotavg_l1_step(rel, n, kind=1, rotations=R, **opts)
        if D["not_pd"]:
            S["termination"] = 2
            break
        R = full(D)
        S["irls_iterations"] += 1
        if D["xmax"] <= opts.get("tolerance", 1e-5):
            S["termination"] = 0
            break
    return S, R


def _to_views(D, n):
    R = np.zeros((n, 3, 3))
    R[D["view_ids"]] = D["rotations"]
    return R


@pytest.mark.parametrize("name", ["complete32", "banded65"])
def test_chained_steps_are_the_solver(gpu_ctx, name):
    rel, n, thr, _, _ = _scene(gpu_ctx, name)
    opts = dict(max_angular_error_deg=thr)
    S, R = _chain(gpu_ctx, rel, n, opts)
    rg, vg, _, _, Sg = gpu_ctx.rotation_averaging_l1(rel, n, **opts)
    for k in S:
        assert Sg[k] == S[k], (k, Sg[k], S[k])
    assert np.array_equal(rg, R)
    print("\n%s chained: %s" % (name, S))


def test_not_positive_definite_path(gpu_ctx):
    """kind 2 with zero weight on every edge of one view: its rows of the Laplacians are zero, the flag is set and no
    direction is returned; a following well-posed solve on the same scratch clears the flag (d_scal[0] is zeroed on
    every solve) and matches the reference's weighted least-squares step."""
    rel, n, thr, D0, _ = _scene(gpu_ctx, "complete32")
    sc = sr.Scene.from_device(D0)
    rng = np.random.default_rng(4)
    w = rng.uniform(0.5, 2.0, sc.nr)
    v = rng.standard_normal(sc.nr)
    w0 = w.copy()
    view = 5
    for e, (a, b) in enumerate(sc.ab):
        if view in (a, b):
            w0[3 * e:3 * e + 3] = 0.0
    D = gpu_ctx.debug_rotavg_l1_step(rel, n, kind=2, weights=[w0, w, w0, w], rhs=[v, v, v, v], max_angular_error_deg=thr)
    assert D["sys_not_pd"].tolist() == [True, False, True, False]
    assert np.isnan(D["dx"][0]).all() and np.isnan(D["dx"][2]).all() and np.isfinite(D["dx"][1]).all()
    assert np.array_equal(D["dx"][1], D["dx"][3])
    lap = D["laplacians"][0]
    assert not lap[:, view - 1, :].any() and not lap[:, :sc.n, view - 1].any()
    L, Lm = sc.laplacian(w)
    q = {"laplacian": max(sr._ratio(D["laplacians"][1][k, :sc.n], L[k], Lm[k]) for k in range(3)),
         "bwd": max(sr.backward_error(D["laplacians"][1][k, :sc.n], D["dx"][1].reshape(3, sc.n)[k], D["laplacians"][1][k, sc.n])
                    for k in range(3)) / U}
    H = (sc.At @ sp.diags(w) @ sc.A).tocsc()
    dx = scipy.sparse.linalg.spsolve(H, sc.At @ v)
    assert np.abs(dx - D["dx"][1]).max() <= 1e-10 * np.abs(dx).max()
    assert not sr.over_bar(q, {}, sc), q


def test_invalid_states(gpu_ctx, r3dlib):
    rel, n, thr, D0, _ = _scene(gpu_ctx, "complete33")
    st = D0["state0"]

    def with_(i, j, v):
        s = [a.copy() for a in st]
        s[i][j] = v
        return s

    b = D0["b"]
    bad = [with_(0, 2, np.nan), with_(5, 0, np.inf), with_(3, 4, 0.0), with_(4, 1, -1.0),
           with_(2, 7, abs(b[7]) * 0.5 - 1e-300),  # u below |A x - b|: f2 or f1 >= 0
           [a[:-1] if i == 2 else a for i, a in enumerate(st)]]
    for s in bad:
        with pytest.raises(r3dlib.R3DError) as e:
            gpu_ctx.debug_rotavg_l1_step(rel, n, state=s, tau=D0["tau0"], max_angular_error_deg=thr)
        assert e.value.code == -1
    for tau in (0.0, -1.0, np.nan, np.inf):
        with pytest.raises(r3dlib.R3DError) as e:
            gpu_ctx.debug_rotavg_l1_step(rel, n, state=st, tau=tau, max_angular_error_deg=thr)
        assert e.value.code == -1
    with pytest.raises(r3dlib.R3DError):
        gpu_ctx.debug_rotavg_l1_step(rel, n, kind=3)
