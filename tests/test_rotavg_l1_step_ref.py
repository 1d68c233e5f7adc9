"""The reference of one L1 rotation-averaging step (rotavg_l1_step_ref) on the CPU: its Newton step solves the unreduced
KKT system, its float64 values agree with the exact ones within their own c u A, the restatement's steps
(rotavg_l1_ref.l1_regression) pass its bars along their whole trajectory, and the bars reject plausible kernel slips."""
import numpy as np
import pytest
from fractions import Fraction
from scipy.spatial.transform import Rotation

import rotavg_l1_ref as ref
import rotavg_l1_step_ref as sr
from rotavg_scenes import complete_edges, make_problem


def component_major(v):
    """(m, 3) per view, row 0 the held view -> 3n component-major."""
    return np.asarray(v)[1:].T.ravel()


def trace_step(sc, b, t):
    """One traced l1_regression iteration as (state, tau, a step dict in r3d_debug_rotavg_l1_step's layout)."""
    st = (component_major(t["x"]), t["Ax"].ravel(), t["u"].ravel(), t["lam1"].ravel(), t["lam2"].ravel(),
          component_major(t["Atv"]))
    d = (component_major(t["dx"]), t["Adx"].ravel(), t["du"].ravel(), t["dlam1"].ravel(), t["dlam2"].ravel(),
         component_major(t["Atdv"]))
    return st, t["tau"], d


def restatement_trajectory(sc, b):
    tr = []
    ref.l1_regression(sc.ab, b.reshape(-1, 3), sc.m, trace=tr.append)
    return tr


@pytest.fixture(scope="module")
def small():
    """An 11-view complete graph with 20 % gross outliers kept (threshold 180 degrees), at its spanning-tree start."""
    m = 11
    rel, _, _ = make_problem(m, complete_edges(m), noise_deg=0.5, outlier_frac=0.2, seed=5)
    _, _, _, _, ab, Rab, views = ref.kept_problem(rel, m, 180.0)
    sc = sr.Scene(len(views), ab, Rab)
    R0 = ref.spanning_tree_start(ab, Rab, sc.m)
    b = ref.residuals(ab, Rab, R0).ravel()
    return sc, b, R0, restatement_trajectory(sc, b)


def _states(tr):
    return [0, len(tr) // 2, len(tr) - 1]


def test_newton_step_solves_the_unreduced_kkt_system(small):
    """The sparse unreduced solve leaves a residual at rounding level, its Schur complement onto x is A^T diag(sigma) A,
    and the reduced system (Laplacians, right-hand sides) gives the same dx."""
    sc, b, _, tr = small
    for which in (0, len(tr) // 2):
        st, tau, _ = trace_step(sc, b, tr[which])
        K = sr.KKT(sc, b, st, tau)
        d = K.solve()
        rx, mx, rr, mr = K.kkt_residual(*d)
        assert np.abs(rx).max() <= 1e-12 * mx.max() and (np.abs(rr) <= 1e-12 * mr).all()
        J, _, _ = K.jacobian()
        J = J.toarray()
        nv = sc.nv
        S = -J[:nv, nv:] @ np.linalg.solve(J[nv:, nv:], J[nv:, :nv])
        L, _, r, _ = K.reduced()
        for k in range(3):
            blk = slice(k * sc.n, (k + 1) * sc.n)
            assert np.abs(S[blk, blk] - L[k]).max() <= 1e-11 * np.abs(L[k]).max()
            # no coupling between components
            assert np.abs(np.delete(S[blk], np.r_[blk], axis=1)).max() <= 1e-11 * np.abs(L[k]).max()
            dxk = np.linalg.solve(L[k], r[k])
            assert np.abs(dxk - d[0][blk]).max() <= 1e-10 * np.abs(dxk).max()


@pytest.mark.parametrize("which", [0, "mid", "late"])
def test_float64_reference_agrees_with_exact(small, which):
    """Laplacians, right-hand sides, sdg and |F_tau|^2 of the float64 reference within c u A of the exact values, and
    the emulated solve within c u kappa |x| of the exact solution of the systems it factored."""
    sc, b, _, tr = small
    i = {0: 0, "mid": len(tr) // 2, "late": len(tr) - 1}[which]
    st, tau, _ = trace_step(sc, b, tr[i])
    K = sr.KKT(sc, b, st, tau)
    L, Lm, r, A_r = K.reduced()
    D = sr.emulate_pd(sc, b, st, tau)
    E = sr.exact(sc, b, st, tau, D["laplacians"])
    c = sr.bars(sc)
    n = sc.n
    for k in range(3):
        err = np.array([[float(abs(Fraction(L[k][i2, j]) - E["lap"][k][i2][j])) for j in range(n)] for i2 in range(n)])
        assert (err <= c["laplacian"] * sr.U * Lm[k]).all()
        err = np.array([float(abs(Fraction(r[k][j]) - E["lap"][k][n][j])) for j in range(n)])
        assert (err <= c["rhs"] * sr.U * A_r[k]).all(), (err / (sr.U * A_r[k])).max()
        xs = np.array([float(v) for v in E["x"][k]])
        kappa = np.linalg.cond(D["laplacians"][k, :n])
        assert np.abs(D["dx"].reshape(3, n)[k] - xs).max() <= 16 * n * sr.U * kappa * np.abs(xs).max()
    sdg, res, A_sdg, A_sq = K.norms()
    assert abs(Fraction(sdg) - E["sdg"]) <= c["sdg"] * sr.U * A_sdg
    assert abs(Fraction(res) ** 2 - E["sq"]) <= c["resnorm"] * sr.U * A_sq
    assert (np.abs(L) <= Lm * (1 + 1e-12)).all() and (np.abs(r) <= A_r * (1 + 1e-12)).all()


def test_restatement_steps_pass_the_bars(small):
    """Every Newton step of rotavg_l1_ref.l1_regression, start to stop, is within the bars of the reference at the
    state it started from: this pins the restatement the end-to-end GPU tests compare against."""
    sc, b, _, tr = small
    worst = {}
    for t in tr:
        st, tau, d = trace_step(sc, b, t)
        D = dict(zip(("dx", "Adx", "du", "dl1", "dl2", "Atdv"), d), not_pd=False, accepted=t["accepted"])
        K = sr.KKT(sc, b, st, tau)
        f1, f2 = K.f1, K.f2
        rmin = sr.ratio_test(f1, f2, K.l1, K.l2, *d[1:5])
        D.update(rmin=rmin, step_max=float(rmin.min()), resnorm0=K.norms()[1])
        D["trials"] = [(s, K.trial(*d, s)[1][1]) for s in t["steps"]]
        q, ex = sr.check_pd(D, sc, b, st, tau)
        ex.pop("trials")  # the restatement's own norms are numpy's, not the reference's
        bad = sr.over_bar(q, ex, sc)
        assert not bad, bad
        for k, v in q.items():
            worst[k] = max(worst.get(k, 0.0), v)
    print("\nrestatement vs reference over %d steps: %s" % (len(tr), worst))


@pytest.mark.parametrize("mutant", [m for m in sr.MUTANTS if m not in sr.IRLS_MUTANTS])
def test_bars_reject_each_pd_mutant(small, mutant):
    """The emulated step passes; with one slip it fails a ratio by more than 10 times its bar, or a decision."""
    sc, b, _, tr = small
    c = sr.bars(sc)
    for i in (0, len(tr) - 1):
        st, tau, _ = trace_step(sc, b, tr[i])
        q, ex = sr.check_pd(sr.emulate_pd(sc, b, st, tau), sc, b, st, tau)
        assert not sr.over_bar(q, ex, sc)
        q, ex = sr.check_pd(sr.emulate_pd(sc, b, st, tau, mutate=(mutant,)), sc, b, st, tau)
        far = [k for k, v in q.items() if v > 10 * c[k.replace("_new", "")]]
        assert far or not all(ex.values()), (mutant, q, ex)


def test_bars_reject_the_irls_mutant(small):
    sc, b, _, _ = small
    c = sr.bars(sc)
    q, ex = sr.check_irls(sr.emulate_irls(sc, b, 5.0), sc, 5.0)
    assert not sr.over_bar(q, ex, sc), q
    q, _ = sr.check_irls(sr.emulate_irls(sc, b, 5.0, mutate=("irls_weight_power",)), sc, 5.0)
    assert q["w"] > 10 * c["w"]
    # and the reference's weighted least-squares step is the solution of the emulated systems
    D = sr.emulate_irls(sc, b, 5.0)
    dx = sr.Irls(sc, b, 5.0).solve()
    assert np.abs(dx - D["dx"]).max() <= 1e-12 * np.abs(dx).max()


@pytest.mark.parametrize("angle", [1e-9, 1e-3, 1.0, np.pi - 1e-3, np.pi - 1e-6])
def test_log_and_exp_against_known_rotation_vectors(angle):
    """The Ceres log (rotavg_l1_ref.R_to_aa, the device's formula) and scipy's both return a known rotation vector
    within the reference's bar, near 0 and near pi; exp by Ceres' formula, Taylor branch included, matches scipy."""
    rng = np.random.default_rng(3)
    c = sr.bars(sr.Scene(2, [[0, 1]], np.eye(3)[None]))["b"]
    for _ in range(20):
        ax = rng.standard_normal(3)
        w = ax / np.linalg.norm(ax) * angle
        Q = Rotation.from_rotvec(w).as_matrix()
        sc = sr.Scene(2, [[0, 1]], Q[None])
        got, A = sr.residuals(sc, np.stack([np.eye(3), np.eye(3)]))
        assert sr._ratio(got, w, A) <= c
        assert sr._ratio(ref.R_to_aa(Q), w, A) <= c
    for th in (1e-9, 1e-7, 0.3):
        x = rng.standard_normal(3)
        x *= th / np.linalg.norm(x)
        assert np.abs(ref.aa_to_R(x) - Rotation.from_rotvec(x).as_matrix()).max() <= 2 * sr.U
