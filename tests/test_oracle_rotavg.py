"""CPU: the rotation-averaging oracle (oracle_rotavg.cpp) against independent code -- brute-force triangle lists with
numpy angles, networkx's 2-edge-connected components, numpy.linalg.eigh, the ground truth of noise-free scenes and
scipy.optimize.least_squares on the same residual -- and the library's host-only component filter on matches."""
import itertools

import networkx as nx
import numpy as np
import pytest
from scipy.optimize import least_squares
from scipy.spatial.transform import Rotation

from oracle import pyoracle_rotavg as rpo
from rotavg_scenes import (angle_deg, axis_angle, banded_ring, complete_edges, gauge_error_fro, make_problem,
                           random_rotation)


def _canonical(rel):
    """(ij (E,2) with i < j, R_ij (E,3,3)) of the OK records."""
    ok = rel["status"] == 0
    I, J, R = rel["I"][ok], rel["J"][ok], rel["rotation"][ok]
    ij = np.c_[np.minimum(I, J), np.maximum(I, J)]
    Rc = np.array([R[k] if I[k] < J[k] else R[k].T for k in range(len(I))])
    return ij, Rc


def _largest_2ec(G):
    comps = [sorted(c) for c in nx.k_edge_components(G, 2) if len(c) >= 2]
    if not comps:
        return set()
    return set(max(comps, key=lambda c: (len(c), -c[0])))


def test_triplets_match_brute_force():
    rng = np.random.default_rng(3)
    n = 14
    edges = [e for e in complete_edges(n) if rng.random() < 0.6]
    rel, Rs, _ = make_problem(n, edges, noise_deg=1.5, outlier_frac=0.25, seed=4, outlier_min_deg=8.0)
    ij, R = _canonical(rel)
    tri, err, valid = rpo.triplets(ij, R, n)
    idx = {tuple(e): k for k, e in enumerate(ij.tolist())}
    exp = {}
    for i, j, k in itertools.combinations(range(n), 3):
        if (i, j) in idx and (j, k) in idx and (i, k) in idx:
            cyc = R[idx[(i, k)]].T @ R[idx[(j, k)]] @ R[idx[(i, j)]]
            exp[(i, j, k)] = angle_deg(cyc)
    got = {tuple(t): (float(e), bool(v)) for t, e, v in zip(tri.tolist(), err, valid)}
    assert set(got) == set(exp) and len(exp) > 50
    margin = min(abs(a - 5.0) for a in exp.values())
    assert margin > 1e-3, "scene too close to the threshold for a numpy cross-check"
    for t, a in exp.items():
        assert abs(got[t][0] - a) < 1e-4, t
        assert got[t][1] == (a < 5.0), t
    assert 0 < sum(v for _, v in got.values()) < len(got)


def _graph_cases():
    rng = np.random.default_rng(8)
    cases = []
    # two dense clusters joined by a bridge, a pendant view, an isolated pair
    a = [(i, j) for i in range(6) for j in range(i + 1, 6)]
    b = [(i, j) for i in range(6, 11) for j in range(i + 1, 11)]
    cases.append((14, a + b + [(5, 6), (10, 11), (12, 13)]))
    # equal clusters: the tie keeps the one with the smaller view id
    cases.append((8, [(0, 1), (1, 2), (0, 2), (5, 6), (6, 7), (5, 7), (2, 5)]))
    # a chain of cycles with bridges between them, parallel edges, random sparse graphs
    cases.append((9, [(0, 1), (1, 2), (2, 0), (2, 3), (3, 4), (4, 5), (5, 6), (6, 3), (6, 7), (7, 8), (8, 7)]))
    for t in range(6):
        n = int(rng.integers(10, 40))
        E = [(int(i), int(j)) for i, j in itertools.combinations(range(n), 2) if rng.random() < 3.0 / n]
        cases.append((n, E))
    cases.append((5, [(0, 1), (1, 2), (2, 3)]))  # a tree: no component
    return cases


@pytest.mark.parametrize("case", range(10))
def test_components_match_networkx(case, r3dlib):
    n, E = _graph_cases()[case]
    G = nx.MultiGraph()
    G.add_nodes_from(range(n))
    G.add_edges_from(E)
    if len(set(map(tuple, map(sorted, E)))) == len(E):
        exp = _largest_2ec(nx.Graph(G))
    else:  # parallel edges (k_edge_components wants a simple graph): cycles {0,1,2}, {3,4,5,6} and the 2-cycle {7,8}
        exp = {3, 4, 5, 6}
    got = rpo.largest_biedge_component(np.array(E, np.uint32).reshape(-1, 2), n)
    assert set(np.nonzero(got)[0].tolist()) == exp
    # the library's host-only filter on a PairWiseMatches with these pairs
    pairs = np.array(E, np.uint32).reshape(-1, 2)
    ofs = np.arange(len(pairs) + 1, dtype=np.uint64)
    m = np.zeros(len(pairs), r3dlib.indmatch_dtype)
    m["i"] = np.arange(len(pairs))
    mm = r3dlib.Matches.from_csr(pairs, ofs, m)
    kept = mm.keep_largest_biedge_component().to_dict()
    exp_pairs = {(int(i), int(j)) for i, j in pairs if int(i) in exp and int(j) in exp}
    assert set(kept) == exp_pairs
    src = mm.to_dict()
    for k, v in kept.items():
        assert np.array_equal(v, src[k])


def test_linear_subspace_matches_eigh():
    rel, Rs, _ = make_problem(25, banded_ring(25, 3), noise_deg=2.0, seed=5)
    ij, R = _canonical(rel)
    M, Q, it = rpo.l2_subspace(ij, R, 25)
    assert 0 < it < 100
    # M built independently: block rows [R_ab | -I]
    A = np.zeros((3 * len(ij), 75))
    for e, (a, b) in enumerate(ij):
        A[3 * e:3 * e + 3, 3 * a:3 * a + 3] = R[e]
        A[3 * e:3 * e + 3, 3 * b:3 * b + 3] = -np.eye(3)
    Mn = A.T @ A
    sigma = 1e-7 * 6
    assert np.allclose(M, Mn + sigma * np.eye(75), atol=1e-12)
    w, V = np.linalg.eigh(Mn)
    assert w[3] - w[2] > 1e-3
    P = V[:, :3] @ V[:, :3].T
    assert np.abs(Q @ Q.T - P).max() <= 1e-9
    assert np.abs(Q.T @ Q - np.eye(3)).max() <= 1e-12


@pytest.mark.parametrize("refine", [False, True])
def test_noise_free_recovers_truth(refine):
    n = 30
    rel, Rs, _ = make_problem(n, [e for e in complete_edges(n) if (e[1] - e[0]) % 4 != 2], seed=11)
    rot, vk, ek, sup, s = rpo.rotation_averaging(rel, n + 2, refine=refine)
    assert s["success"] == 1 and ek.all() and vk[:n].all() and not vk[n:].any()
    assert (sup > 0).all() and s["n_valid_triplets"] == s["n_triplets"]
    assert np.array_equal(rot[vk.nonzero()[0][0]], np.eye(3))
    assert gauge_error_fro(rot, Rs, vk) <= 1e-10
    assert not rot[n:].any()


def _scipy_refine(ij, R, R0):
    m = len(R0)
    x0 = np.concatenate([Rotation.from_matrix(r).as_rotvec() for r in R0])

    def fun(x):
        Rm = Rotation.from_rotvec(x.reshape(-1, 3)).as_matrix()
        out = []
        for e, (a, b) in enumerate(ij):
            out.append(Rotation.from_matrix(R[e].T @ Rm[b] @ Rm[a].T).as_rotvec())
        return np.concatenate(out)

    r = least_squares(fun, x0, method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=20000)
    return Rotation.from_rotvec(r.x.reshape(m, 3)).as_matrix(), 0.5 * float(r.fun @ r.fun)


def test_refinement_matches_scipy_least_squares():
    n = 20
    rel, Rs, _ = make_problem(n, complete_edges(n), noise_deg=2.0, seed=13)
    rot0, vk, _, _, _ = rpo.rotation_averaging(rel, n, refine=False)
    rot, vk, ek, _, s = rpo.rotation_averaging(rel, n, refine=True, function_tolerance=1e-14, gradient_tolerance=1e-14,
                                               parameter_tolerance=1e-14)
    assert s["lm_termination"] in (1, 2, 3) and s["lm_final_cost"] < s["lm_initial_cost"]
    ij, R = _canonical(rel)
    Rsp, cost = _scipy_refine(ij, R, rot0)
    assert abs(s["lm_final_cost"] - cost) <= 1e-8 * cost
    for a, b in ij:
        assert np.abs(rot[b] @ rot[a].T - Rsp[b] @ Rsp[a].T).max() <= 1e-7


def test_outliers_are_rejected():
    n = 24
    rel, Rs, out = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.1, seed=17)
    assert out.sum() > 10
    rot, vk, ek, sup, s = rpo.rotation_averaging(rel, n)
    assert not ek[out].any() and ek[~out].all()
    assert s["n_kept_edges"] == (~out).sum() and s["n_kept_views"] == n
    assert np.degrees(gauge_error_fro(rot, Rs, vk) / np.sqrt(2)) < 1.0


def test_ring_without_triangles_fails_softly():
    n = 12
    rel, _, _ = make_problem(n, banded_ring(n, 1), seed=2)
    rot, vk, ek, sup, s = rpo.rotation_averaging(rel, n)
    assert s["success"] == 0 and s["n_triplets"] == 0 and not vk.any() and not ek.any() and not rot.any()


def test_invalid_inputs():
    rel, _, _ = make_problem(5, complete_edges(5), seed=1)
    bad = rel.copy()
    bad[0]["J"] = bad[0]["I"]
    with pytest.raises(rpo.OracleError) as e:
        rpo.rotation_averaging(bad, 5)
    assert e.value.code == -1
    with pytest.raises(rpo.OracleError) as e:
        rpo.rotation_averaging(rel, 4)
    assert e.value.code == -1
    dup = np.concatenate([rel, rel[:1]])
    dup[-1]["I"], dup[-1]["J"] = rel[0]["J"], rel[0]["I"]
    with pytest.raises(rpo.OracleError) as e:
        rpo.rotation_averaging(dup, 5)
    assert e.value.code == -1
    dup[-1]["status"] = 3  # not an edge: ignored
    assert rpo.rotation_averaging(dup, 5)[4]["n_edges"] == len(rel)
    with pytest.raises(rpo.OracleError) as e:
        rpo.rotation_averaging(rel, 5, method=1)
    assert e.value.code == -5


def test_cycle_error_threshold_is_strict_float():
    """Triangles one float ulp either side of 5 degrees: the decision is float(error) < 5.0f."""
    Ri = np.eye(3)
    ax = np.array([0.3, -0.5, 0.8])
    lo, hi = 4.999, 5.001
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        if rpo.cycle_error(Ri, Ri, axis_angle(ax, mid)) < np.float32(5.0):
            lo = mid
        else:
            hi = mid
    below = rpo.cycle_error(Ri, Ri, axis_angle(ax, lo))
    above = rpo.cycle_error(Ri, Ri, axis_angle(ax, hi))
    assert np.float32(below) == np.nextafter(np.float32(5.0), np.float32(0)) and np.float32(above) == np.float32(5.0)
