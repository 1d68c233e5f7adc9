"""CPU: the translation-averaging oracle (oracle_transavg.cpp) against independent code -- the ground truth of noise-free
scenes, the KKT conditions of the convex soft-L1 problem with scipy.optimize.least_squares unable to improve on its
optimum, scipy.optimize.least_squares on the chordal problem from the oracle's start, networkx's 2-edge-connected components, finite differences of the Jacobian and the soft-L1 corrector."""
import networkx as nx
import numpy as np
import pytest
from scipy.optimize import least_squares

from oracle import pyoracle_transavg as pto
from transavg_scenes import aligned_error, banded_ring, complete_edges, make_problem, similarity_align

M64 = (1 << 64) - 1


def _start_value(k):
    """The chordal start draw (splitmix64, uniform in [0, 1)), written out independently."""
    z = (k * 0x9E3779B97F4A7C15 + 0x6A09E667F3BCC909) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    z ^= z >> 31
    return (z >> 11) / float(1 << 53)


def _edges(rel):
    """(I, J, unit t_IJ) of the records in their stored orientation."""
    t = rel["translation"] / np.linalg.norm(rel["translation"], axis=1, keepdims=True)
    return rel["I"].astype(int), rel["J"].astype(int), t


@pytest.mark.parametrize("method", [pto.TRANSAVG_L2_CHORDAL, pto.TRANSAVG_SOFTL1])
@pytest.mark.parametrize("graph", ["complete", "ring"])
def test_noise_free_recovers_the_truth(method, graph):
    n = 25 if graph == "complete" else 40
    edges = complete_edges(n) if graph == "complete" else banded_ring(n, 3)
    rel, Rs, Cs, _ = make_problem(n, edges, seed=11)
    # tolerances below the upstream ones: this pins the optimum, not the stopping rule
    C, T, vk, ek, S = pto.translation_averaging(rel, Rs, np.ones(n, bool), n, method=method, gradient_tolerance=1e-16,
                                                function_tolerance=1e-15, parameter_tolerance=1e-14)
    assert S["success"] and vk.all() and ek.all() and S["n_kept_views"] == n and S["n_kept_edges"] == len(edges)
    assert aligned_error(C, Cs, vk) <= 1e-9
    assert not C[0].any()                                    # the gauge: the lowest kept view sits at the origin
    assert np.abs(T + np.einsum("vij,vj->vi", Rs, C)).max() <= 1e-12 * max(1.0, np.abs(T).max())
    assert S["lm_final_cost"] <= 1e-12 * S["lm_initial_cost"]


def _softl1_parts(rel, Rs):
    I, J, u = _edges(rel)
    return I, J, u, np.einsum("eab,ecb->eac", Rs[J], Rs[I])   # R_IJ = R_J R_I^T


def test_softl1_optimum_with_active_bounds():
    """The problem is convex: the oracle's t with the scales that are optimal for it (max(1, (t_J - R_IJ t_I) . u),
    the loss grows with |r|) satisfies the KKT conditions, some scales sit on the bound, and scipy's least_squares
    (soft_l1 on the scalar residual |r_e| with f_scale = a is the same cost) started there finds nothing lower."""
    n, a = 10, 0.01
    rel, Rs, Cs, _ = make_problem(n, complete_edges(n), noise_deg=1.0, seed=12, scale_range=(0.5, 3.0))
    C, T, vk, _, S = pto.translation_averaging(rel, Rs, np.ones(n, bool), n, method=pto.TRANSAVG_SOFTL1, function_tolerance=1e-15,
                                               parameter_tolerance=1e-14, max_iterations=5000)
    I, J, u, Rij = _softl1_parts(rel, Rs)
    q = T[J] - np.einsum("eab,eb->ea", Rij, T[I])
    s = np.maximum(1.0, (q * u).sum(1))
    active = s == 1.0
    assert active.any() and (~active).any()                  # the bound holds some scales and not others
    r = q - s[:, None] * u
    sq = (r * r).sum(1)
    rho1 = 1.0 / np.sqrt(1.0 + sq / (a * a))
    assert abs(0.5 * (2 * a * a * (np.sqrt(1 + sq / (a * a)) - 1)).sum() - S["lm_final_cost"]) <= 1e-10 * S["lm_final_cost"]
    g = np.zeros((n, 3))
    np.add.at(g, J, rho1[:, None] * r)
    np.add.at(g, I, -np.einsum("eba,eb->ea", Rij, rho1[:, None] * r))
    ref = np.abs(rho1[:, None] * r).sum()
    assert np.abs(g[1:]).max() <= 1e-7 * ref                 # stationary in t (t_0 is held)
    gs = -(rho1[:, None] * r * u).sum(1)                     # d cost / d s_e
    assert np.abs(gs[~active]).max() <= 1e-7 * ref and (gs[active] >= -1e-7 * ref).all()

    def resid(p):
        t = np.vstack([np.zeros(3), p[:3 * (n - 1)].reshape(-1, 3)])
        rr = t[J] - np.einsum("eab,eb->ea", Rij, t[I]) - p[3 * (n - 1):, None] * u
        return np.linalg.norm(rr, axis=1)

    p0 = np.concatenate([T[1:].ravel(), s])
    lb = np.concatenate([np.full(3 * (n - 1), -np.inf), np.ones(len(s))])
    sol = least_squares(resid, p0, loss="soft_l1", f_scale=a, bounds=(lb, np.inf), xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=200)
    assert sol.cost >= S["lm_final_cost"] * (1 - 1e-9)


def test_chordal_matches_scipy_from_the_same_start():
    n = 12
    rel, Rs, Cs, _ = make_problem(n, complete_edges(n), noise_deg=1.0, seed=13)
    C, _, vk, _, S = pto.translation_averaging(rel, Rs, np.ones(n, bool), n, function_tolerance=1e-15, parameter_tolerance=1e-14,
                                               max_iterations=5000)
    I, J, t = _edges(rel)
    u = -np.einsum("eba,eb->ea", Rs[J], t)                   # -R_J^T t_IJ

    def resid(p):
        X = np.vstack([np.zeros(3), p.reshape(-1, 3)])
        d = X[J] - X[I]
        return (d / np.linalg.norm(d, axis=1, keepdims=True) - u).ravel()

    p0 = np.array([_start_value(k) for k in range(3 * (n - 1))])
    sol = least_squares(resid, p0, method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=20000)
    X = np.vstack([np.zeros(3), sol.x.reshape(-1, 3)])
    assert abs(S["lm_final_cost"] - sol.cost) <= 1e-8 * sol.cost
    # the chordal cost does not see the scale: compare the shapes
    assert aligned_error(C, X, vk) <= 1e-7 and aligned_error(C, Cs, vk) < 0.05


def test_kept_component_matches_networkx():
    # views 0..9 dense, 10..15 dense, bridge (9, 10), pendant 16 on 3; 17..19 without edges; view 5 not rotation-kept;
    # a record that is not OK and one with edge_use = 0
    e = [(i, j) for i in range(10) for j in range(i + 1, 10)] + [(i, j) for i in range(10, 16) for j in range(i + 1, 16)]
    e += [(9, 10), (3, 16), (16, 17)]
    rel, Rs, Cs, _ = make_problem(20, e, noise_deg=0.3, seed=14)
    rel["status"][1] = pto.RELPOSE_NO_MODEL
    use = np.ones(len(rel), bool)
    use[2] = False
    rk = np.ones(20, bool)
    rk[5] = False
    C, T, vk, ek, S = pto.translation_averaging(rel, Rs, rk, 20, method=pto.TRANSAVG_SOFTL1, edge_use=use)
    usable = (rel["status"] == 0) & use & rk[rel["I"]] & rk[rel["J"]]
    G = nx.Graph()
    G.add_edges_from(zip(rel["I"][usable].tolist(), rel["J"][usable].tolist()))
    comps = [sorted(c) for c in nx.k_edge_components(G, 2) if len(c) >= 2]
    best = set(max(comps, key=lambda c: (len(c), -c[0])))
    assert set(np.nonzero(vk)[0].tolist()) == best
    assert S["n_edges"] == usable.sum()
    exp_e = usable & np.isin(rel["I"], list(best)) & np.isin(rel["J"], list(best))
    assert np.array_equal(ek, exp_e) and S["n_kept_edges"] == exp_e.sum()
    assert not C[~vk].any() and not T[~vk].any()


@pytest.mark.parametrize("method", [pto.TRANSAVG_L2_CHORDAL, pto.TRANSAVG_SOFTL1])
def test_jacobian_matches_finite_differences(method):
    rng = np.random.default_rng(15)
    for _ in range(5):
        xi, xj = rng.normal(size=3), rng.normal(size=3) * 3
        s = 1.0 + rng.random()
        ed = np.concatenate([rng.normal(size=3) * 0.8, rng.normal(size=3)])
        ed[3:] /= np.linalg.norm(ed[3:])
        r, J = pto.edge(method, xi, xj, s, ed)
        p = np.concatenate([xi, xj, [s]])
        h = 1e-6
        for k in range(7 if method == pto.TRANSAVG_SOFTL1 else 6):
            dp = np.zeros(7)
            dp[k] = h
            rp, _ = pto.edge(method, (p + dp)[:3], (p + dp)[3:6], (p + dp)[6], ed)
            rm, _ = pto.edge(method, (p - dp)[:3], (p - dp)[3:6], (p - dp)[6], ed)
            assert np.abs((rp - rm) / (2 * h) - J[:, k]).max() <= 1e-7 * max(1.0, np.abs(J).max())
        if method == pto.TRANSAVG_SOFTL1:   # the residual itself, with an independent rotation matrix
            th = np.linalg.norm(ed[:3])
            K = np.array([[0, -ed[2], ed[1]], [ed[2], 0, -ed[0]], [-ed[1], ed[0], 0]]) / th
            R = np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K
            assert np.abs(r - (xj - R @ xi - s * ed[3:])).max() <= 1e-12
        else:
            d = xj - xi
            assert np.abs(r - (d / np.linalg.norm(d) - ed[:3])).max() <= 1e-15 * 10


def test_softl1_corrector():
    a = 0.01
    for sq in (0.0, 1e-6, 1e-4, 0.3, 25.0):
        rho, rho1 = pto.softl1_rho(sq, a)
        b = a * a
        assert abs(rho - 2 * b * (np.sqrt(1 + sq / b) - 1)) <= 1e-15 * max(1.0, rho)
        assert abs(rho1 - 1 / np.sqrt(1 + sq / b)) <= 1e-15
        h = max(sq, 1e-6) * 1e-5
        lo = max(sq - h, 0.0)
        fd = (pto.softl1_rho(sq + h, a)[0] - pto.softl1_rho(lo, a)[0]) / (sq + h - lo)
        assert abs(fd - rho1) <= 1e-6 * rho1


def test_invalid_inputs_and_l1():
    rel, Rs, _, _ = make_problem(5, complete_edges(5), seed=16)
    rk = np.ones(5, bool)
    bad = rel.copy()
    bad[0]["J"] = bad[0]["I"]
    dup = np.concatenate([rel, rel[:1]])
    dup[-1]["I"], dup[-1]["J"] = rel[0]["J"], rel[0]["I"]
    zero = rel.copy()
    zero[1]["translation"] = 0.0
    nan = rel.copy()
    nan[2]["translation"][0] = np.nan
    for r, n in ((bad, 5), (rel, 4), (dup, 5), (zero, 5), (nan, 5)):
        with pytest.raises(pto.OracleError) as e:
            pto.translation_averaging(r, Rs, rk, n)
        assert e.value.code == -1
    with pytest.raises(pto.OracleError) as e:
        pto.translation_averaging(rel, Rs, rk, 5, method=pto.TRANSAVG_L1)
    assert e.value.code == -5
    # an unusable duplicate is not an error once edge_use drops it... but an unused zero translation is ignored
    use = np.ones(len(zero), bool)
    use[1] = False
    pto.translation_averaging(zero, Rs, rk, 5, edge_use=use)


def test_similarity_align_is_exact():
    rng = np.random.default_rng(17)
    X = rng.normal(size=(20, 3))
    th = 0.7
    R = np.array([[np.cos(th), -np.sin(th), 0], [np.sin(th), np.cos(th), 0], [0, 0, 1]])
    Y = 2.5 * X @ R.T + np.array([1.0, -2.0, 3.0])
    assert np.abs(similarity_align(X, Y) - Y).max() <= 1e-12
