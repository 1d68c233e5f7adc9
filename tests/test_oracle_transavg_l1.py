"""CPU restatement of the L-infinity translation LP (transavg_l1_ref) against HiGHS on an LP built independently here:
the optimal value gamma*, the feasibility of the returned point, lambda >= 1 and convergence; the noise-free scene
recovers the truth."""
import numpy as np
import pytest
import scipy.sparse as sp
from scipy.optimize import linprog

import transavg_l1_ref as ref
from oracle import pyoracle_transavg as pto
from transavg_scenes import aligned_error, banded_ring, complete_edges, make_problem


def highs_gamma(rel, Rs, edge_kept, view_kept):
    """gamma* by HiGHS.  Columns: T of every kept view (the lowest one fixed at 0 by its bounds), one lambda per kept
    record, gamma; rows: +-(T_J - R_J R_I^T T_I - lambda u) - gamma <= 0."""
    recs = np.nonzero(edge_kept)[0]
    views = np.nonzero(view_kept)[0]
    col = {v: 3 * k for k, v in enumerate(views)}
    m, ne = len(views), len(recs)
    nv = 3 * m + ne + 1
    A = sp.lil_matrix((6 * ne, nv))
    for k, e in enumerate(recs):
        i, j = int(rel["I"][e]), int(rel["J"][e])
        Rij = Rs[j] @ Rs[i].T
        t = rel["translation"][e]
        u = t / np.linalg.norm(t)
        for a in range(3):
            for sgn, row in ((1.0, 6 * k + a), (-1.0, 6 * k + 3 + a)):
                A[row, col[j] + a] += sgn
                for b in range(3):
                    A[row, col[i] + b] -= sgn * Rij[a, b]
                A[row, 3 * m + k] = -sgn * u[a]
                A[row, nv - 1] = -1.0
    c = np.zeros(nv)
    c[-1] = 1.0
    bounds = [(0.0, 0.0)] * 3 + [(None, None)] * (3 * m - 3) + [(1.0, None)] * ne + [(None, None)]
    r = linprog(c, A_ub=A.tocsr(), b_ub=np.zeros(6 * ne), bounds=bounds, method="highs")
    assert r.status == 0
    return r.fun


def check_point(rel, Rs, C, T, vk, ek, lam, gamma):
    """The returned point is feasible for the bound gamma: |T_J - R_IJ T_I - lambda u| <= gamma, lambda >= 1, C = -R^T T,
    the gauge view at T = 0."""
    tol = 1e-9 * (1.0 + gamma)
    e = np.nonzero(ek)[0]
    I, J = rel["I"][e].astype(int), rel["J"][e].astype(int)
    u = rel["translation"][e] / np.linalg.norm(rel["translation"][e], axis=1, keepdims=True)
    r = T[J] - np.einsum("eab,ecb,ec->ea", Rs[J], Rs[I], T[I]) - lam[e][:, None] * u
    assert np.abs(r).max() <= gamma + tol
    assert lam[e].min() >= 1.0 - tol and not lam[~ek].any()
    assert np.allclose(C[vk], -np.einsum("vba,vb->va", Rs[vk], T[vk]), rtol=0, atol=1e-12 * max(1.0, np.abs(T).max()))
    assert not T[np.nonzero(vk)[0][0]].any()


SCENES = {
    "complete30": lambda: (30, make_problem(30, complete_edges(30), noise_deg=0.5, seed=5)),
    "ring60": lambda: (60, make_problem(60, banded_ring(60, 3), noise_deg=0.5, seed=5)),
    "outliers": lambda: (30, make_problem(30, complete_edges(30), noise_deg=0.5, outlier_frac=0.05, seed=8)),
    "scales": lambda: (30, make_problem(30, complete_edges(30), noise_deg=1.0, seed=6, scale_range=(0.3, 3.0))),
}


@pytest.mark.parametrize("scene", list(SCENES))
def test_optimal_value_matches_highs(scene):
    n, (rel, Rs, _, _) = SCENES[scene]()
    C, T, vk, ek, lam, S = ref.translation_averaging_l1(rel, Rs, np.ones(n, bool), n)
    assert S["success"] and S["termination"] == 0 and S["n_kept_views"] == n
    g_h = highs_gamma(rel, Rs, ek, vk)
    assert abs(S["gamma"] - g_h) <= 1e-9 * max(1.0, g_h), (S["gamma"], g_h)
    check_point(rel, Rs, C, T, vk, ek, lam, S["gamma"])
    assert S["max_primal_violation"] <= 1e-9 * (1.0 + S["gamma"])
    if scene == "scales":
        assert (lam[ek] < 1.0 + 1e-6).any()  # the bound lambda >= 1 is active for some edges


def test_noise_free_recovers_the_truth():
    n = 40
    rel, Rs, Cs, _ = make_problem(n, complete_edges(n), seed=5)
    C, T, vk, ek, lam, S = ref.translation_averaging_l1(rel, Rs, np.ones(n, bool), n)
    assert S["termination"] == 0
    assert S["gamma"] <= 1e-8
    assert aligned_error(C, Cs, vk) < 1e-8


def test_lp_rows_are_the_residual():
    """build_lp's G y - h on a random point equals the L-infinity rows written out edge by edge."""
    n = 12
    rel, Rs, _, _ = make_problem(n, complete_edges(n), noise_deg=1.0, seed=9)
    vk, ek = np.ones(n, bool), np.ones(len(rel), bool)
    G, h, c, views, recs = ref.build_lp(rel, Rs, vk, ek)
    rng = np.random.default_rng(0)
    y = rng.standard_normal(G.shape[1])
    T = np.vstack([np.zeros(3), y[:3 * (n - 1)].reshape(-1, 3)])
    lam, gam = y[3 * (n - 1):-1], y[-1]
    I, J = rel["I"].astype(int), rel["J"].astype(int)
    u = rel["translation"] / np.linalg.norm(rel["translation"], axis=1, keepdims=True)
    r = T[J] - np.einsum("eab,ecb,ec->ea", Rs[J], Rs[I], T[I]) - lam[:, None] * u
    exp = np.hstack([r - gam, -r - gam, (1.0 - lam)[:, None]])
    assert np.allclose((G @ y - h).reshape(-1, 7), exp, rtol=0, atol=1e-12)
    assert c[-1] == 1.0 and not c[:-1].any()


def test_invalid_inputs_and_bad_options():
    """The library's validation, restated: bad records fail with -1 (the oracle's edge checks), bad options with
    ValueError before any work."""
    rel, Rs, _, _ = make_problem(5, complete_edges(5), seed=36)
    rk = np.ones(5, bool)
    bad = rel.copy()
    bad[0]["J"] = bad[0]["I"]
    dup = np.concatenate([rel, rel[:1]])
    dup[-1]["I"], dup[-1]["J"] = rel[0]["J"], rel[0]["I"]
    zero = rel.copy()
    zero[1]["translation"] = 0.0
    inf = rel.copy()
    inf[2]["translation"][1] = np.inf
    for r, n in ((bad, 5), (rel, 4), (dup, 5), (zero, 5), (inf, 5)):
        with pytest.raises(pto.OracleError) as e:
            ref.translation_averaging_l1(r, Rs, rk, n)
        assert e.value.code == -1
    for kw in ({"max_iterations": 0}, {"tolerance": 0.0}, {"tolerance": -1e-9}, {"tolerance": float("nan")}):
        with pytest.raises(ValueError):
            ref.translation_averaging_l1(rel, Rs, rk, 5, **kw)
    *_, S = ref.translation_averaging_l1(rel, Rs, rk, 5, max_iterations=2)
    assert S["termination"] == 1 and S["iterations"] == 2
