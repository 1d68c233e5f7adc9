"""The reference of one L1 translation-averaging iteration (transavg_l1_step_ref) on the CPU: its float64 values agree
with the exact ones within their own c u A, chained steps reproduce the restatement's trajectory (transavg_l1_ref),
and the bars the GPU step test uses reject deliberately wrong variants of the reference."""
import numpy as np
import pytest

import transavg_l1_ref as ref
import transavg_l1_step_ref as sr
from transavg_scenes import complete_edges, make_problem


def scene_from_records(rel, Rs, rk, n, edge_use=None):
    """The kept edges in record order (the restatement's), as the kernels would see them."""
    vk, ek, _ = ref.kept_edges(rel, Rs, rk, n, edge_use)
    views, recs = np.nonzero(vk)[0], np.nonzero(ek)[0]
    local = np.full(n, -1)
    local[views] = np.arange(len(views))
    I, J = rel["I"][recs].astype(int), rel["J"][recs].astype(int)
    R = np.asarray(Rs, np.float64).reshape(-1, 3, 3)
    Rij = np.einsum("eab,ecb->eac", R[J], R[I])
    t = rel["translation"][recs]
    u = t / np.linalg.norm(t, axis=1, keepdims=True)
    return sr.Scene(len(views), np.stack([local[I], local[J]], 1), Rij, u, recs), vk, ek


def trajectory(sc, rel, Rs, vk, ek, max_iterations=100):
    """The restatement's states (y, lambda, s, z) per iteration, on sc's edges (record order)."""
    G, h, c, _, _ = ref.build_lp(rel, Rs, vk, ek)
    states = []

    def keep(it, y, s, z):
        states.append((np.r_[y[:sc.nt], y[-1]], y[sc.nt:sc.nt + sc.ne], s, z))

    _, S = ref.solve(G, h, c, sc.nt, max_iterations=max_iterations, trace=keep)
    return states, S


@pytest.fixture(scope="module")
def small():
    m = 11
    rel, Rs, _, _ = make_problem(m, complete_edges(m), noise_deg=0.5, seed=31)
    sc, vk, ek = scene_from_records(rel, Rs, np.ones(m, bool), m)
    states, S = trajectory(sc, rel, Rs, vk, ek)
    return sc, states, S


def test_scene_stores_both_orientations(small):
    sc, _, _ = small
    assert (sc.ij[:, 0] > sc.ij[:, 1]).any() and (sc.ij[:, 0] < sc.ij[:, 1]).any()


def test_start_point_is_the_restatements(small):
    sc, states, _ = small
    for a, b in zip(sr.start_state(sc), states[0]):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("which", [0, 8, -3])
def test_float64_reference_agrees_with_exact(small, which):
    """Matrix, right-hand side and norms of the float64 reference within c u A of the exact values, at the start and
    at a middle and a late state."""
    from fractions import Fraction
    sc, states, _ = small
    st = states[which]
    R = sr.Step(sc, *st)
    E = sr.exact(sc, st)
    b = sr.bars(sc)
    M = np.array([[float(v) for v in row] for row in E["Mred"]])
    err = np.array([[abs(Fraction(R.Mred[i, j]) - E["Mred"][i][j]) for j in range(sc.N)] for i in range(sc.N)], float)
    assert (err <= b["matrix"] * sr.U * R.A_Mred).all(), np.nanmax(err / (sr.U * R.A_Mred))
    assert np.allclose(M, R.Mred, rtol=0, atol=1e-9 * np.abs(M).max())
    s, z = st[2], st[3]
    Rp = R.rhs(s * z, np.abs(s * z))
    err = np.array([abs(Fraction(Rp["red"][i]) - E["rhs"][i]) for i in range(sc.N)], float)
    assert (err <= b["rhs_pred"] * sr.U * Rp["A_red"]).all()
    nv, nA = R.norms()
    for i in range(5):
        assert abs(Fraction(nv[i]) - E["norms"][i]) <= b["norms"] * sr.U * nA[i], i
    # the magnitudes bound what they stand for
    assert (np.abs(R.Mred) <= R.A_Mred * (1 + 1e-12)).all() and (np.abs(Rp["red"]) <= Rp["A_red"] * (1 + 1e-12)).all()


def test_emulated_step_passes_its_bars_and_solves_exactly(small):
    """The float64 emulation of the library's step passes every bar at a late state, and its direction is within
    c u kappa |x| of the exact solution of the scaled system."""
    sc, states, _ = small
    st = states[-3]
    D = sr.emulate(sc, st)
    q, ex, info = sr.check(D, sc, st)
    assert not sr.over_bar(q, ex, sc, info["allow"]), sr.over_bar(q, ex, sc, info["allow"])
    E = sr.exact(sc, st, D["A"], D["retries"])
    xs = np.array([float(v) for v in E["xs"]])
    got = info["solutions"]["pred"][0]
    assert np.abs(got - xs).max() <= 16 * sc.N * sr.U * E["kappa"] * np.abs(xs).max()


def test_chained_reference_steps_follow_the_restatement(small):
    """Chaining the emulated step from the start point reproduces transavg_l1_ref.solve's trajectory to rounding and
    stops at the same iteration."""
    sc, states, S = small
    st = states[0]
    it = 0
    while True:
        D = sr.emulate(sc, st)
        if D["converged"]:
            break
        st = D["state"]
        it += 1
        want = states[it]
        for a, b in zip(st, want):
            assert np.abs(a - b).max() <= 1e-6 * max(1.0, np.abs(b).max()), it
    assert it == S["iterations"] == len(states) - 1


@pytest.mark.parametrize("mutant", sr.MUTANTS)
def test_bars_reject_each_mutant(small, mutant):
    """A step computed right (the emulation) checked against a deliberately wrong reference is over a bar: the bars
    are tight enough to catch a kernel that makes the same mistake."""
    sc, states, _ = small
    for st in (states[0], states[-3]):
        D = sr.emulate(sc, st)
        q, ex, info = sr.check(D, sc, st)
        assert not sr.over_bar(q, ex, sc, info["allow"])
        q, ex, info = sr.check(D, sc, st, mutate=(mutant,))
        assert sr.over_bar(q, ex, sc, info["allow"]), (mutant, q)
