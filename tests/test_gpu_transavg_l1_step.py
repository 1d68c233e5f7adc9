"""-m gpu: one iteration of r3d_translation_averaging_l1 (r3d_debug_transavg_l1_step: the phases the solver runs per
iteration) against the LP-built reference of transavg_l1_step_ref.py, at the start point and at late states of the
restatement's trajectory (transavg_l1_ref.solve), on scenes whose N = 3 (m - 1) + 1 sits on and across the 32-row tiles
of dense_cholesky, the bench problem (44 850 edges: the grid-stride loops of the one-CTA reductions), a scene with a
bridge, a pendant and unusable records, and one whose view 0 is not rotation-kept.

Each value is held to |gpu - ref| <= c u A (A: the same sum over absolute values; c in transavg_l1_step_ref.bars, a
small multiple of the longest sum), the solves to their normwise backward error on the scaled reduced system and on the
dual equation of the unreduced Newton system, and the step lengths and the update bit for bit.  On scenes of at most
12 views the matrix, right-hand side and norms are also held to their exact values and the predictor's direction to the
exact solution of the scaled system the library factored.  Chained steps reproduce translation_averaging_l1 bit for
bit, which ties the summary's certificate (dual objective, residual norms) to a host recomputation.

The all-retries-failed exit (termination 2) is not exercised: G^T D G is positive semidefinite, an exactly zero column
recovers on the first retry (tested below), and no finite state with s > 0, z >= 0 is known to reach it."""
import numpy as np
import pytest

import transavg_l1_ref as ref
import transavg_l1_step_ref as sr
from fractions import Fraction
from transavg_scenes import banded_ring, complete_edges, make_problem

pytestmark = pytest.mark.gpu
U = sr.U


def _bridge():
    e = [(i, j) for i in range(10) for j in range(i + 1, 10)] + [(i, j) for i in range(10, 16) for j in range(i + 1, 16)]
    e += [(9, 10), (3, 16)]
    rel, Rs, _, _ = make_problem(20, e, noise_deg=0.3, seed=33)
    rel["status"][1] = 3  # RELPOSE_NO_MODEL
    use = np.ones(len(rel), bool)
    use[2] = False
    rk = np.ones(20, bool)
    rk[4] = False
    return rel, Rs, rk, 20, use


def _gauge_not_zero():
    rel, Rs, _, _ = make_problem(14, complete_edges(14), noise_deg=0.5, seed=41)
    rk = np.ones(14, bool)
    rk[0] = False
    return rel, Rs, rk, 14, None


def _complete(m, seed):
    return lambda: (*make_problem(m, complete_edges(m), noise_deg=0.5, seed=seed)[:2], np.ones(m, bool), m, None)


SCENES = {
    "complete11": _complete(11, 51),   # N = 31: the right-hand side row inside the last 32-row tile
    "complete12": _complete(12, 52),   # N = 34: across it
    "complete22": _complete(22, 53),   # N = 64: the right-hand side row in a tile of its own
    "complete60": _complete(60, 31),   # test_gpu_transavg_l1.py's complete graph
    "ring200": lambda: (*make_problem(200, banded_ring(200, 3), noise_deg=0.5, seed=32)[:2], np.ones(200, bool), 200, None),
    "bench300": _complete(300, 7),
    "bridge_pendant_unusable": _bridge,
    "gauge_not_view0": _gauge_not_zero,
}
_cache = {}


def _scene(name):
    """(inputs, restatement states in record order and their kept records / views, its summary)."""
    if name not in _cache:
        rel, Rs, rk, n, use = SCENES[name]()
        vk, ek, _ = ref.kept_edges(rel, Rs, rk, n, use)
        G, h, c, views, recs = ref.build_lp(rel, Rs, vk, ek)
        nt = 3 * (len(views) - 1)
        states = []
        _, S = ref.solve(G, h, c, nt, trace=lambda it, y, s, z: states.append((y, s, z)))
        _cache[name] = ((rel, Rs, rk, n, use), states, views, recs, nt, S)
    return _cache[name]


def _device_state(D, st, views, recs, nt):
    """A restatement state in the library's order: kept edges by their records, T by local view id."""
    assert np.array_equal(D["view_ids"], views)
    perm = np.searchsorted(recs, D["edge_record"])
    assert np.array_equal(recs[perm], D["edge_record"])
    y, s, z = st
    lam = y[nt:-1]
    return (np.r_[y[:nt], y[-1]], lam[perm].copy(), s.reshape(-1, 7)[perm].ravel().copy(), z.reshape(-1, 7)[perm].ravel().copy())


def _states(name):
    """The start point and late states: half way, and 4 and 2 iterations before the restatement stops (past its
    regularised factorisations near the optimum)."""
    _, states, _, _, _, _ = _scene(name)
    n = len(states)
    return [None] + sorted({n // 2, n - 5, n - 3})


def _step(ctx, name, which):
    (rel, Rs, rk, n, use), states, views, recs, nt, _ = _scene(name)
    D0 = ctx.debug_transavg_l1_step(rel, Rs, rk, n, edge_use=use)
    if which is None:
        return D0, D0["state0"]
    st = _device_state(D0, states[which], views, recs, nt)
    return ctx.debug_transavg_l1_step(rel, Rs, rk, n, edge_use=use, state=st), st


def _exact_checks(D, sc, st):
    """Against the exact values (Fractions): matrix entries, predictor right-hand side, norms, and the predictor's
    direction within c u kappa |x| of the exact solution of the system factored (refined once when regularised)."""
    E = sr.exact(sc, st, D["A"], D["retries"])
    R = sr.Step(sc, *st)
    b = sr.bars(sc)
    N = sc.N
    out = {}
    low = np.tril(np.ones((N, N), bool))
    low[:N - 1, :N - 1] = True
    err = np.array([[float(abs(Fraction(D["A"][i, j]) - E["Mred"][i][j])) if low[i, j] else 0.0 for j in range(N)] for i in range(N)])
    out["x_matrix"] = float((err / np.maximum(U * R.A_Mred, 1e-300)).max())
    Rp = R.rhs(st[2] * st[3], np.abs(st[2] * st[3]))
    err = np.array([float(abs(Fraction(D["A"][N, i]) - E["rhs"][i])) for i in range(N)])
    out["x_rhs"] = float((err / np.maximum(U * Rp["A_red"], 1e-300)).max())
    nv, nA = R.norms()
    out["x_norms"] = max(float(abs(Fraction(D["norms"][i]) - E["norms"][i])) / (U * nA[i]) for i in range(5))
    xs = np.array([float(v) for v in E["xs"]])
    got = D["pred"]["dy"] / D["sc"]
    out["x_forward"] = float(np.abs(got - xs).max() / (U * E["kappa"] * np.abs(xs).max()))
    lim = {"x_matrix": b["matrix"], "x_rhs": b["rhs_pred"], "x_norms": b["norms"], "x_forward": 16.0 * N}
    return out, ["%s %.3g > %.3g" % (k, v, lim[k]) for k, v in out.items() if not v <= lim[k]]


def _fmt(q):
    return " ".join("%s %.3g" % kv for kv in q.items())


@pytest.mark.parametrize("name", list(SCENES))
def test_step_equals_reference(gpu_ctx, name):
    """Every output of one iteration at the start point and at late states against the reference."""
    bad, retried = [], []
    for which in _states(name):
        D, st = _step(gpu_ctx, name, which)
        assert not D["converged"] and not D["failed"]
        sc = sr.Scene.from_device(D)
        if which is None:
            # the start point: s = h - G y computed on the host in the library's order, bit for bit
            for a, b in zip(D["state0"], sr.start_state(sc)):
                assert np.array_equal(a, b)
        q, ex, info = sr.check(D, sc, st)
        bad += ["%s@%s: %s" % (name, which, b) for b in sr.over_bar(q, ex, sc, info["allow"])]
        if sc.m <= 12:
            qx, bx = _exact_checks(D, sc, st)
            q.update(qx)
            bad += ["%s@%s: %s" % (name, which, b) for b in bx]
        if D["retries"]:
            retried.append((which, D["retries"]))
        assert D["not_pd"][:D["retries"]] == [True] * D["retries"] and not D["not_pd"][D["retries"]]
        print("\n%s state %s (N %d, ne %d, retries %d): %s" % (name, which, sc.N, sc.ne, D["retries"], _fmt(q)))
    print("%s: states with retries %s" % (name, retried))
    assert not bad, bad
    if name in ("complete60", "bench300"):
        assert retried  # H100: state 25 of complete60 and state 52 of bench300 each took 3 retries


def test_zero_column_is_retried_once(gpu_ctx):
    """z = 0 on rows 0..5 of every edge incident to one view makes that view's column of the reduced system exactly 0:
    the first factorisation fails, the first retry (1e-18 max diag added) succeeds, the view's direction is exactly 0,
    and the rest is held to the reference's solve of the regularised system."""
    name = "complete12"
    (rel, Rs, rk, n, use), _, _, _, _, _ = _scene(name)
    D0 = gpu_ctx.debug_transavg_l1_step(rel, Rs, rk, n, edge_use=use)
    y, lam, s, z = D0["state0"]
    z = z.copy()
    v = 5
    for e, (I, J) in enumerate(D0["edge_ij"]):
        if v in (I, J):
            z[7 * e:7 * e + 6] = 0.0
    D = gpu_ctx.debug_transavg_l1_step(rel, Rs, rk, n, edge_use=use, state=(y, lam, s, z))
    cols = slice(3 * (v - 1), 3 * v)
    N = D["N"]
    assert not D["A"][:N, cols].any() and not D["A"][cols, :].any() and not D["A"][N, cols].any()
    assert D["not_pd"][:2] == [True, False] and D["retries"] == 1 and not D["failed"]
    # the predictor's right-hand side of the view is 0 too (wt = 0 where z = 0), so is its direction; the corrector's
    # is not (sigma mu / s), and its direction there is that over the added diagonal
    assert not D["pred"]["dy"][cols].any() and not D["A"][N, cols].any()
    sc = sr.Scene.from_device(D)
    st = (y, lam, s, z)
    q, ex, info = sr.check(D, sc, st)
    bad = sr.over_bar(q, ex, sc, info["allow"])
    print("\nzero column: %s" % _fmt(q))
    assert not bad, bad
    E = sr.exact(sc, st, D["A"], D["retries"])
    xs = np.array([float(x) for x in E["xs"]])
    got = D["pred"]["dy"] / D["sc"]
    keep = np.ones(N, bool)
    keep[cols] = False
    # kappa of the regularised system is 1e18 from the zero column alone; the rest is held to kappa of its own block
    Mf = sr.regularised(sr.scaled_system(D["A"])[0], 1)[np.ix_(keep, keep)]
    assert np.abs(got - xs)[keep].max() <= 16 * N * U * np.linalg.cond(Mf) * np.abs(xs).max()


@pytest.mark.parametrize("name", ["complete22", "complete60"])
def test_chained_steps_are_the_solver(gpu_ctx, name):
    """k debug steps from the start point give translation_averaging_l1(max_iterations=k) bit for bit (T, lambda,
    gamma) for k = 1, 2, 10 and to convergence; the converged state's norms, recomputed on the host, match the
    summary's certificate within c u A."""
    (rel, Rs, rk, n, use), _, _, _, _, _ = _scene(name)
    D = gpu_ctx.debug_transavg_l1_step(rel, Rs, rk, n, edge_use=use)
    chain = [D["state0"]]
    while not D["converged"]:
        assert not D["failed"] and len(chain) <= 100
        chain.append(D["state"])
        D = gpu_ctx.debug_transavg_l1_step(rel, Rs, rk, n, edge_use=use, state=D["state"])
    views, recs = D["view_ids"], D["edge_record"]
    for k in (1, 2, 10, len(chain) - 1):
        C, T, vk, ek, lam, S = gpu_ctx.translation_averaging_l1(rel, Rs, rk, n, edge_use=use, max_iterations=max(k, 1))
        y, l_, _, _ = chain[k]
        assert S["iterations"] == k
        assert np.array_equal(T[views[1:]].ravel(), y[:-1]) and not T[views[0]].any()
        assert np.array_equal(lam[recs], l_)
        assert S["gamma"] == y[-1]
    assert S["termination"] == 0
    sc = sr.Scene.from_device(D)
    nv, nA = sr.Step(sc, *chain[-1]).norms()
    c = sr.bars(sc)["norms"]
    assert np.array_equal(D["norms"][[4, 2, 1]], [S["dual_objective"], S["max_dual_violation"], S["max_primal_violation"]])
    for i, k in ((4, "dual_objective"), (2, "max_dual_violation"), (1, "max_primal_violation")):
        assert abs(S[k] - nv[i]) <= c * U * nA[i], (k, S[k], nv[i])
    print("\n%s: %d iterations chained, certificate %s" % (name, len(chain) - 1,
                                                          _fmt({k: abs(S[k] - nv[i]) / (U * nA[i]) for i, k in
                                                                ((4, "dual_objective"), (2, "max_dual_violation"),
                                                                 (1, "max_primal_violation"))})))


def test_invalid_states(gpu_ctx, r3dlib):
    (rel, Rs, rk, n, use), _, _, _, _, _ = _scene("complete11")
    D = gpu_ctx.debug_transavg_l1_step(rel, Rs, rk, n, edge_use=use)
    y, lam, s, z = D["state0"]
    nan_y = y.copy()
    nan_y[3] = np.nan
    s0 = s.copy()
    s0[10] = 0.0
    zneg = z.copy()
    zneg[4] = -1e-300
    for st in ((y, lam[:-1], s, z), (y[:-1], lam, s, z), (y, lam, s, np.r_[z, 1.0]), (nan_y, lam, s, z), (y, lam, s0, z),
               (y, lam, s, zneg)):
        with pytest.raises(r3dlib.R3DError) as e:
            gpu_ctx.debug_transavg_l1_step(rel, Rs, rk, n, edge_use=use, state=st)
        assert e.value.code == -1
