"""-m gpu: r3d_translation_averaging_l1 against the CPU restatement (transavg_l1_ref) and HiGHS: success, counts, kept
sets, iterations and termination identical, both converged, gamma within 2e-9 (1 + gamma) of the restatement's, centres,
translations and edge scales within 1e-8 of the scene's scale, the returned point feasible;
repeated calls bit-identical; and the chain relative poses -> rotations -> L1 translations -> structure -> bundle
adjustment on a synthetic ring.

The optimal point of the LP is in general not unique (gamma* is).  Where a factorisation near the optimum needs the
regularisation fallback on either side, the two stop at different points of the optimal face; those scenes state their
measured distance and a bar beside it."""
import numpy as np
import pytest

import transavg_l1_ref as ref
from oracle import pyoracle_transavg as pto
from regard3d_b200 import synth
from relpose_scenes import ring_truth
from test_oracle_transavg_l1 import check_point, highs_gamma
from transavg_scenes import aligned_error, banded_ring, complete_edges, make_problem

pytestmark = pytest.mark.gpu


def _compare(gpu_ctx, rel, Rs, rk, n, point_tol=1e-8, iteration_tol=0, **kw):
    """point_tol: centres and translations within point_tol of the scene's scale, lambda within point_tol, where some
    factorisation fell back to regularisation on either side (otherwise 1e-8).  Near the optimum the regularised
    directions are those in which the optimal face is flat, so there the two solvers may stop at different optimal
    points; gamma agrees regardless."""
    got = gpu_ctx.translation_averaging_l1(rel, Rs, rk, n, **kw)
    exp = ref.translation_averaging_l1(rel, Rs, rk, n, **kw)
    Cg, Tg, vg, eg, lg, Sg = got
    Co, To, _, _, lo, Sr = exp
    scale = max(np.abs(Co).max(), np.abs(To).max(), 1e-300)
    print("gpu: %d iterations (%d regularised), gamma %.15g; cpu: %d iterations (%d regularised), gamma %.15g; "
          "max |dC|, |dT| / scale %.3g %.3g, max |d lambda| %.3g" % (
              Sg["iterations"], Sg["regularized_factorizations"], Sg["gamma"], Sr["iterations"], Sr["regularized_factorizations"],
              Sr["gamma"], np.abs(Cg - Co).max() / scale, np.abs(Tg - To).max() / scale, np.abs(lg - lo).max()))
    for k in ("success", "n_edges", "n_kept_edges", "n_kept_views"):
        assert Sg[k] == Sr[k], (k, Sg[k], Sr[k])
    assert np.array_equal(vg, exp[2]) and np.array_equal(eg, exp[3])
    if not Sr["success"]:
        assert not Cg.any() and not Tg.any() and not lg.any() and Sg["termination"] == -1
        return got, exp
    assert Sg["termination"] == 0 and Sr["termination"] == 0
    assert abs(Sg["iterations"] - Sr["iterations"]) <= iteration_tol
    assert abs(Sg["gamma"] - Sr["gamma"]) <= 2e-9 * (1.0 + Sr["gamma"])
    tol = point_tol if Sg["regularized_factorizations"] or Sr["regularized_factorizations"] else 1e-8
    assert np.abs(Cg - Co).max() <= tol * scale and np.abs(Tg - To).max() <= tol * scale
    assert np.abs(lg - lo).max() <= tol
    assert abs(Sg["gamma"] - Sg["dual_objective"]) <= 1e-9 * (1.0 + Sg["gamma"])
    assert Sg["max_primal_violation"] <= 1e-9 * (1.0 + Sg["gamma"]) and Sg["max_dual_violation"] <= 1e-9
    check_point(rel, Rs, Cg, Tg, vg, eg, lg, Sg["gamma"])
    assert Sg["ms_solve"] > 0 and Sg["ms_device_total"] >= Sg["ms_solve"]
    return got, exp


def test_complete_graph(gpu_ctx):
    # H100: 27 iterations on both sides, 3 / 6 regularised factorisations, points 1.3e-5 of the scale apart, lambda 1.2e-3
    n = 60
    rel, Rs, Cs, _ = make_problem(n, complete_edges(n), noise_deg=0.5, seed=31)
    (C, _, vk, _, _, S), _ = _compare(gpu_ctx, rel, Rs, np.ones(n, bool), n, point_tol=1e-2)
    assert S["success"] and S["n_kept_views"] == n
    assert aligned_error(C, Cs, vk) < 0.05


def test_bench_problem(gpu_ctx):
    """scripts/bench_transavg_l1.py's problem: 300 views, 44 850 edges.  H100: 52 iterations against the restatement's
    54, 9 / 8 regularised factorisations, gamma equal to 1e-15, points 1.8e-3 of the scale apart, lambda 0.1."""
    n = 300
    rel, Rs, Cs, _ = make_problem(n, complete_edges(n), noise_deg=0.5, seed=7)
    (C, _, vk, _, _, S), _ = _compare(gpu_ctx, rel, Rs, np.ones(n, bool), n, point_tol=0.5, iteration_tol=3)
    assert S["success"] and S["n_kept_views"] == n


def test_banded_ring(gpu_ctx):
    n = 200
    rel, Rs, _, _ = make_problem(n, banded_ring(n, 3), noise_deg=0.5, seed=32)
    # H100: 19 iterations on both sides, 3 regularised factorisations each, points 1.8e-8 of the scale apart
    (_, _, _, _, _, S), _ = _compare(gpu_ctx, rel, Rs, np.ones(n, bool), n, point_tol=1e-6)
    assert S["n_kept_views"] == n


def test_bridge_pendant_unusable_records(gpu_ctx):
    # as test_gpu_transavg: two dense groups joined by a bridge, a pendant view, views without edges, a record that is
    # not OK, one with edge_use = 0 and a view that rotation averaging did not keep
    e = [(i, j) for i in range(10) for j in range(i + 1, 10)] + [(i, j) for i in range(10, 16) for j in range(i + 1, 16)]
    e += [(9, 10), (3, 16)]
    rel, Rs, _, _ = make_problem(20, e, noise_deg=0.3, seed=33)
    rel["status"][1] = pto.RELPOSE_NO_MODEL
    use = np.ones(len(rel), bool)
    use[2] = False
    rk = np.ones(20, bool)
    rk[4] = False
    (C, T, vk, ek, lam, S), _ = _compare(gpu_ctx, rel, Rs, rk, 20, edge_use=use)
    assert set(np.nonzero(vk)[0].tolist()) == set(range(10)) - {4}
    assert not C[~vk].any() and not T[~vk].any() and not ek[1] and not ek[2] and not lam[~ek].any()
    # the same kept sets as the other translation methods
    _, _, vo, eo, _ = pto.translation_averaging(rel, Rs, rk, 20, edge_use=use)
    assert np.array_equal(vk, vo) and np.array_equal(ek, eo)


def test_outliers_against_highs(gpu_ctx):
    n = 40
    rel, Rs, _, _ = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.05, seed=38)
    (_, _, vk, ek, _, S), _ = _compare(gpu_ctx, rel, Rs, np.ones(n, bool), n)
    g_h = highs_gamma(rel, Rs, ek, vk)
    assert abs(S["gamma"] - g_h) <= 1e-9 * max(1.0, g_h), (S["gamma"], g_h)


def test_no_component(gpu_ctx):
    rel, Rs, _, _ = make_problem(4, [(0, 1), (1, 2), (2, 3)], seed=39)  # a path: no bi-edge-connected component
    _compare(gpu_ctx, rel, Rs, np.ones(4, bool), 4)


def test_repeated_calls_are_bit_identical(gpu_ctx):
    n = 50
    rel, Rs, _, _ = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.05, seed=35)
    a = gpu_ctx.translation_averaging_l1(rel, Rs, np.ones(n, bool), n)
    b = gpu_ctx.translation_averaging_l1(rel, Rs, np.ones(n, bool), n)
    for x, y in zip(a[:5], b[:5]):
        assert np.array_equal(x, y)
    for k in ("iterations", "termination", "gamma", "dual_objective", "max_primal_violation", "max_dual_violation"):
        assert a[5][k] == b[5][k]


def test_iteration_cap(gpu_ctx):
    n = 30
    rel, Rs, _, _ = make_problem(n, complete_edges(n), noise_deg=0.5, seed=5)
    *_, S = gpu_ctx.translation_averaging_l1(rel, Rs, np.ones(n, bool), n, max_iterations=3)
    assert S["termination"] == 1 and S["iterations"] == 3


def test_invalid_inputs(gpu_ctx, r3dlib):
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
    for r, n, kw in ((bad, 5, {}), (rel, 4, {}), (dup, 5, {}), (zero, 5, {}), (inf, 5, {}), (rel, 5, {"max_iterations": 0}),
                     (rel, 5, {"tolerance": 0.0}), (rel, 5, {"tolerance": -1e-9}), (rel, 5, {"tolerance": float("nan")})):
        with pytest.raises(r3dlib.R3DError) as e:
            gpu_ctx.translation_averaging_l1(r, Rs, rk, n, **kw)
        assert e.value.code == -1, kw
    # the LM entry point still refuses the L1 method
    with pytest.raises(r3dlib.R3DError) as e:
        gpu_ctx.translation_averaging(rel, Rs, rk, 5, method=r3dlib.TRANSAVG_L1)
    assert e.value.code == -5


def test_two_devices_equal_one(r3dlib):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    n = 40
    rel, Rs, _, _ = make_problem(n, complete_edges(n), noise_deg=0.5, seed=37)
    c1, c2 = r3dlib.Context((0,)), r3dlib.Context((0, 1))
    a = c1.translation_averaging_l1(rel, Rs, np.ones(n, bool), n)
    b = c2.translation_averaging_l1(rel, Rs, np.ones(n, bool), n)
    for x, y in zip(a[:5], b[:5]):
        assert np.array_equal(x, y)
    c1.close()
    c2.close()


def test_end_to_end_relative_poses_to_bundle_adjustment(gpu_ctx, r3dlib):
    """match_pairs -> relative_poses -> rotation_averaging -> translation_averaging_l1 -> SfmData with these poses ->
    tracks of the AC-RANSAC inliers -> structure_from_tracks -> remove_outliers -> sfm_bundle_adjust on an 8-view ring."""
    n = 8
    sc = synth.make_scene(n, 1500, 64, "msurf", seed=61)
    pairs = synth.exhaustive_pairs(n)
    gpu_ctx.clear_regions()
    for v in range(n):
        gpu_ctx.upload_regions(v, sc["descs"][v], sc["xys"][v])
    put = gpu_ctx.match_pairs(pairs, 0.8)
    Ks = np.array([[1.1 * max(int(w), int(h)), w / 2.0, h / 2.0] for w, h in zip(sc["widths"], sc["heights"])])
    rel, inl = gpu_ctx.relative_poses(put, sc["widths"], sc["heights"], Ks)
    Rg, rk, ek_rot, _, _ = gpu_ctx.rotation_averaging(rel, n)
    (C, T, vk, _, _, S), _ = _compare(gpu_ctx, rel, Rg, rk, n, edge_use=ek_rot)
    assert S["success"] and vk.sum() >= 6
    Rs, ts = ring_truth(n, 1500, 64, "msurf", seed=61)
    Ct = np.array([-np.asarray(R).T @ np.asarray(t) for R, t in zip(Rs, ts)])
    err = aligned_error(C, Ct, vk)
    sd = r3dlib.SfmData()
    sd.add_intrinsic(0, r3dlib.CAM_PINHOLE, sc["w"], sc["h"], Ks[0][0], Ks[0][1], Ks[0][2])
    for v in range(n):
        sd.add_view(v, "image%06d.jpg" % v, sc["w"], sc["h"], id_intrinsic=0, id_pose=v)
        if vk[v]:
            sd.add_pose(v, Rg[v], C[v])
    tracks = r3dlib.Tracks.build(inl, 2)
    gpu_ctx.structure_from_tracks(sd, tracks)
    gpu_ctx.remove_outliers(sd, 4.0, 2, 2.0)
    s = gpu_ctx.sfm_bundle_adjust(sd, max_iterations=50)
    lms = sd.landmarks()
    rms = np.sqrt(2.0 * s["final_cost"] / max(1, sum(len(lm["obs"]) for lm in lms)))
    print("end-to-end L1: centre error %.3g of the diameter, %d landmarks, RMS %.3f px" % (err, len(lms), rms))
    # bars from an H100 run (centre error 3.1e-4 of the diameter, 2245 landmarks, RMS 0.600 px) with the margin of the
    # other translation methods' test
    assert len(lms) > 1000
    assert err < 2e-3
    assert rms < 0.8
