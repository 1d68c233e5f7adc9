"""-m gpu: r3d_rotation_averaging_l1 against its CPU restatement (rotavg_l1_ref.py): the triplet and valid-triplet counts,
edge_support, edge_kept, view_kept and success identical; the L1RA, primal-dual, backtrack and IRLS counts and the
termination identical; rotations within 1e-8 after the gauge."""
import numpy as np
import pytest

import rotavg_l1_ref as ref
from regard3d_b200 import synth
from relpose_scenes import ring_truth
from rotavg_scenes import banded_ring, complete_edges, gauge_error_fro, make_problem

pytestmark = pytest.mark.gpu

COUNTS = ("success", "n_edges", "n_triplets", "n_valid_triplets", "n_kept_edges", "n_kept_views")
ITERS = ("l1_iterations", "pd_iterations", "pd_backtracks", "irls_iterations", "termination")


def _compare(gpu_ctx, rel, n_views, rot_tol=1e-8, **opts):
    got = gpu_ctx.rotation_averaging_l1(rel, n_views, **opts)
    exp = ref.rotation_averaging_l1(rel, n_views, **opts)
    rg, vg, eg, sg, Sg = got
    ro, vo, eo, so, So = exp
    for k in COUNTS:
        assert Sg[k] == So[k], (k, Sg[k], So[k])
    assert np.array_equal(sg, so) and np.array_equal(eg, eo) and np.array_equal(vg, vo)
    if not So["success"]:
        assert not rg.any() and Sg["termination"] == -1
        return got, exp
    for k in ITERS:
        assert Sg[k] == So[k], (k, Sg[k], So[k])
    assert abs(Sg["initial_l1_cost"] - So["initial_l1_cost"]) <= 1e-9 * max(So["initial_l1_cost"], 1e-300)
    assert abs(Sg["final_l1_cost"] - So["final_l1_cost"]) <= 1e-8 * max(So["final_l1_cost"], 1e-300)
    assert np.abs(rg - ro).max() <= rot_tol
    r0 = np.nonzero(vg)[0][0]
    assert np.array_equal(rg[r0], np.eye(3))
    return got, exp


def _deg(R, Rs, kept):
    return np.degrees(gauge_error_fro(R, Rs, kept) / np.sqrt(2))


def test_complete_graph_with_outliers(gpu_ctx):
    n = 60
    rel, Rs, out = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.15, seed=21)
    (rg, vg, eg, _, S), _ = _compare(gpu_ctx, rel, n)
    assert S["success"] and S["n_triplets"] == n * (n - 1) * (n - 2) // 6 and S["termination"] == 0
    assert not eg[out].any() and eg[~out].all()
    assert _deg(rg, Rs, vg) < 0.5
    t = S["ms_triplets"], S["ms_l1"], S["ms_irls"]
    assert all(x > 0 for x in t) and S["ms_device_total"] >= sum(t) * 0.999


def test_banded_ring(gpu_ctx):
    n = 200
    rel, _, _ = make_problem(n, banded_ring(n, 3), noise_deg=0.5, seed=22)
    (_, _, _, _, S), _ = _compare(gpu_ctx, rel, n)
    assert S["n_kept_views"] == n


def test_bridge_pendant_and_views_without_edges(gpu_ctx):
    # as test_gpu_rotavg.py: views 0..9 dense, 10..15 dense, joined by the bridge (9, 10); pendant 16 on 3; views
    # 17..19 have no edges; one record is not OK
    e = [(i, j) for i in range(10) for j in range(i + 1, 10)] + [(i, j) for i in range(10, 16) for j in range(i + 1, 16)]
    e += [(9, 10), (3, 16)]
    rel, _, _ = make_problem(20, e, noise_deg=0.3, seed=23)
    rel = np.concatenate([rel, rel[:1]])
    rel[-1]["status"] = 1
    (rg, vg, eg, sg, _), _ = _compare(gpu_ctx, rel, 20)
    assert set(np.nonzero(vg)[0].tolist()) == set(range(10))
    assert not rg[10:].any() and sg[-1] == 0 and not eg[-1]


def test_bench_problem(gpu_ctx):
    """The 300-view problem of scripts/bench_rotavg_l1.py."""
    n = 300
    rel, Rs, _ = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.1, seed=7, outlier_min_deg=0.0)
    (rg, vg, _, _, S), _ = _compare(gpu_ctx, rel, n)
    assert S["n_kept_views"] == n and S["termination"] == 0 and _deg(rg, Rs, vg) < 0.5


def test_robustness_within_the_cpu_bound(gpu_ctx):
    """test_oracle_rotavg_l1.py's robustness scene (every outlier kept by the triplet test): the GPU result is within
    the bound the CPU restatement is held to there."""
    from test_oracle_rotavg_l1 import ROBUST_L1_BOUND_DEG, robust_scene
    rel, Rs, n = robust_scene()
    (rg, vg, _, _, _), _ = _compare(gpu_ctx, rel, n, max_angular_error_deg=180.0)
    assert _deg(rg, Rs, vg) < ROBUST_L1_BOUND_DEG


def test_repeated_calls_are_bit_identical(gpu_ctx):
    n = 50
    rel, _, _ = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.1, seed=26)
    a = gpu_ctx.rotation_averaging_l1(rel, n)
    b = gpu_ctx.rotation_averaging_l1(rel, n)
    for x, y in zip(a[:4], b[:4]):
        assert np.array_equal(x, y)
    for k in ITERS + ("initial_l1_cost", "final_l1_cost", "n_valid_triplets"):
        assert a[4][k] == b[4][k]


def test_two_devices_equal_one(r3dlib):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    n = 40
    rel, _, _ = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.1, seed=27)
    c1, c2 = r3dlib.Context((0,)), r3dlib.Context((0, 1))
    a, b = c1.rotation_averaging_l1(rel, n), c2.rotation_averaging_l1(rel, n)
    for x, y in zip(a[:4], b[:4]):
        assert np.array_equal(x, y)
    c1.close()
    c2.close()


def test_iteration_caps(gpu_ctx):
    n = 60
    rel, _, _ = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.15, seed=21)
    (_, _, _, _, S), _ = _compare(gpu_ctx, rel, n, l1_max_iterations=1, irls_max_iterations=0)
    assert S["termination"] == 1 and S["l1_iterations"] == 1 and S["irls_iterations"] == 0
    (_, _, _, _, S), _ = _compare(gpu_ctx, rel, n, irls_max_iterations=1)
    assert S["termination"] == 1 and S["irls_iterations"] == 1


def test_no_component(gpu_ctx):
    # a path has no triangle: no edge is supported
    rel, _, _ = make_problem(6, [(i, i + 1) for i in range(5)], noise_deg=0.3, seed=3)
    (rg, vg, eg, sg, S), _ = _compare(gpu_ctx, rel, 6)
    assert S["success"] == 0 and not rg.any() and not vg.any() and not eg.any() and not sg.any()
    assert S["l1_iterations"] == S["pd_iterations"] == S["irls_iterations"] == 0


def test_invalid_inputs_and_options(gpu_ctx, r3dlib):
    rel, _, _ = make_problem(5, complete_edges(5), seed=1)
    bad = rel.copy()
    bad[0]["J"] = bad[0]["I"]
    dup = np.concatenate([rel, rel[:1]])
    dup[-1]["I"], dup[-1]["J"] = rel[0]["J"], rel[0]["I"]
    for args in ((bad, 5), (rel, 4), (dup, 5)):
        with pytest.raises(r3dlib.R3DError) as e:
            gpu_ctx.rotation_averaging_l1(*args)
        assert e.value.code == -1
    for opts in (dict(l1_max_iterations=0), dict(irls_max_iterations=-1), dict(tolerance=0.0), dict(tolerance=float("nan")),
                 dict(irls_sigma_deg=0.0), dict(irls_sigma_deg=float("nan")), dict(max_angular_error_deg=0.0)):
        with pytest.raises(r3dlib.R3DError) as e:
            gpu_ctx.rotation_averaging_l1(rel, 5, **opts)
        assert e.value.code == -1, opts
    # the L2 entry point keeps answering the L1 method with R3D_ERR_UNSUPPORTED
    with pytest.raises(r3dlib.R3DError) as e:
        gpu_ctx.rotation_averaging(rel, 5, method=r3dlib.ROTAVG_L1)
    assert e.value.code == -5


def test_end_to_end_l1_rotations_then_l1_translations(gpu_ctx):
    """Regard3D's L1 + L1 global configuration on an 8-view ring scene: relative_poses, rotation_averaging_l1, then
    translation_averaging_l1 on its kept edges.  The rotations are within 0.5 degrees of synth.make_scene's up to the
    gauge (the relative poses carry the estimation noise of 0.5 px image noise)."""
    n = 8
    sc = synth.make_scene(n, 1500, 64, "msurf", seed=61)
    pairs = synth.exhaustive_pairs(n)
    gpu_ctx.clear_regions()
    for v in range(n):
        gpu_ctx.upload_regions(v, sc["descs"][v], sc["xys"][v])
    put = gpu_ctx.match_pairs(pairs, 0.8)
    Ks = np.array([[1.1 * max(int(w), int(h)), w / 2.0, h / 2.0] for w, h in zip(sc["widths"], sc["heights"])])
    rel, _ = gpu_ctx.relative_poses(put, sc["widths"], sc["heights"], Ks)
    Rs, _ = ring_truth(n, 1500, 64, "msurf", seed=61)
    (rg, vg, eg, _, S), _ = _compare(gpu_ctx, rel, n)
    assert S["success"] and vg.sum() >= 6
    assert _deg(rg, np.asarray(Rs), vg) < 0.5
    cen, tra, tv, te, lam, T = gpu_ctx.translation_averaging_l1(rel, rg, vg, n, edge_use=eg)
    assert T["success"] and T["termination"] == 0 and tv.sum() >= 6 and (lam[te] >= 1.0 - 1e-9).all()
