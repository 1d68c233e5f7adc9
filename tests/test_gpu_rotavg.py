"""-m gpu: r3d_rotation_averaging against the CPU oracle (orc_rotation_averaging): the triplet and valid-triplet counts,
edge_support, edge_kept, view_kept and success identical; refine = 0 rotations within 1e-10; with the refinement the
same LM iteration count, successful steps and termination, the initial cost within 1e-9 and the final cost within 1e-8
relative, rotations within 1e-8 after the gauge."""
import numpy as np
import pytest

from oracle import pyoracle_rotavg as rpo
from regard3d_b200 import synth
from relpose_scenes import ring_truth
from rotavg_scenes import axis_angle, banded_ring, complete_edges, gauge_error_fro, make_problem

pytestmark = pytest.mark.gpu


def _compare(gpu_ctx, rel, n_views, **opts):
    got = gpu_ctx.rotation_averaging(rel, n_views, **opts)
    exp = rpo.rotation_averaging(rel, n_views, **opts)
    rg, vg, eg, sg, Sg = got
    ro, vo, eo, so, So = exp
    for k in ("success", "n_edges", "n_triplets", "n_valid_triplets", "n_kept_edges", "n_kept_views"):
        assert Sg[k] == So[k], (k, Sg[k], So[k])
    assert np.array_equal(sg, so) and np.array_equal(eg, eo) and np.array_equal(vg, vo)
    if not So["success"]:
        assert not rg.any()
        return got, exp
    if not opts.get("refine", True):
        assert Sg["lm_termination"] == -1
        assert np.abs(rg - ro).max() <= 1e-10
        return got, exp
    for k in ("lm_iterations", "lm_successful_steps", "lm_termination"):
        assert Sg[k] == So[k], (k, Sg[k], So[k])
    assert abs(Sg["lm_initial_cost"] - So["lm_initial_cost"]) <= 1e-9 * max(So["lm_initial_cost"], 1e-300)
    assert abs(Sg["lm_final_cost"] - So["lm_final_cost"]) <= 1e-8 * max(So["lm_final_cost"], 1e-300)
    assert np.abs(rg - ro).max() <= 1e-8
    return got, exp


def test_complete_graph_with_outliers(gpu_ctx):
    n = 60
    rel, Rs, out = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.15, seed=21)
    (rg, vg, eg, sg, S), _ = _compare(gpu_ctx, rel, n)
    assert S["success"] and S["n_triplets"] == n * (n - 1) * (n - 2) // 6
    assert not eg[out].any() and eg[~out].all()
    assert np.degrees(gauge_error_fro(rg, Rs, vg) / np.sqrt(2)) < 0.5
    _compare(gpu_ctx, rel, n, refine=False)
    t = S["ms_triplets"], S["ms_init"], S["ms_refine"]
    assert all(x > 0 for x in t) and S["ms_device_total"] >= sum(t) * 0.999


def test_banded_ring(gpu_ctx):
    n = 200
    rel, Rs, _ = make_problem(n, banded_ring(n, 3), noise_deg=0.5, seed=22)
    (rg, vg, _, _, S), _ = _compare(gpu_ctx, rel, n)
    assert S["n_kept_views"] == n
    _compare(gpu_ctx, rel, n, refine=False)


def test_bridge_pendant_and_views_without_edges(gpu_ctx):
    # views 0..9 dense, 10..15 dense, joined by the bridge (9, 10); pendant 16 on 3; views 17..19 have no edges;
    # one record is not OK and one is a 2-view "triangle-free" pair
    e = [(i, j) for i in range(10) for j in range(i + 1, 10)] + [(i, j) for i in range(10, 16) for j in range(i + 1, 16)]
    e += [(9, 10), (3, 16)]
    rel, Rs, _ = make_problem(20, e, noise_deg=0.3, seed=23)
    rel = np.concatenate([rel, rel[:1]])
    rel[-1]["status"] = rpo.RELPOSE_NO_MODEL
    (rg, vg, eg, sg, S), _ = _compare(gpu_ctx, rel, 20)
    assert set(np.nonzero(vg)[0].tolist()) == set(range(10))
    assert not rg[10:].any() and sg[-1] == 0 and not eg[-1]
    _compare(gpu_ctx, rel, 20, refine=False)


def test_threshold_ulps(gpu_ctx):
    """Triangles whose cycle error is one float ulp below 5 degrees, exactly 5.0f and just above: identical decisions."""
    ax = np.array([0.3, -0.5, 0.8])
    I3 = np.eye(3)
    lo, hi = 4.999, 5.001
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        if rpo.cycle_error(I3, I3, axis_angle(ax, mid)) < np.float32(5.0):
            lo = mid
        else:
            hi = mid
    I, J, R = [], [], []
    for t, ang in enumerate([lo, hi, np.nextafter(hi, 10.0), lo - 1e-9, 4.0, 6.0]):
        a, b, c = 3 * t, 3 * t + 1, 3 * t + 2
        I += [a, b, a]
        J += [b, c, c]
        R += [I3, I3, axis_angle(ax, ang)]  # the cycle error is exactly the bisected one
    from regard3d_b200 import capi
    rel = capi.relative_pose_records(I, J, np.array(R))
    got = gpu_ctx.rotation_averaging(rel, 18, refine=False)
    exp = rpo.rotation_averaging(rel, 18, refine=False)
    assert np.array_equal(got[3], exp[3]) and got[4]["n_valid_triplets"] == exp[4]["n_valid_triplets"]
    assert got[4]["n_triplets"] == 6 and exp[4]["n_valid_triplets"] == 3


def test_large_complete_graph_support_is_exact(gpu_ctx):
    n = 400
    rel, Rs, out = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.1, seed=24)
    got = gpu_ctx.rotation_averaging(rel, n, refine=False)
    assert got[4]["n_triplets"] == n * (n - 1) * (n - 2) // 6 >= 10_000_000
    exp = rpo.rotation_averaging(rel, n, refine=False)
    assert np.array_equal(got[3], exp[3]) and got[4]["n_valid_triplets"] == exp[4]["n_valid_triplets"]
    assert np.array_equal(got[2], exp[2]) and np.abs(got[0] - exp[0]).max() <= 1e-10


def test_huber(gpu_ctx):
    n = 40
    rel, Rs, _ = make_problem(n, complete_edges(n), noise_deg=1.0, outlier_frac=0.05, seed=25, outlier_min_deg=3.0)
    (_, _, _, _, S), _ = _compare(gpu_ctx, rel, n, huber_a=0.02)
    assert S["lm_iterations"] > 0


def test_repeated_calls_are_bit_identical(gpu_ctx):
    n = 50
    rel, _, _ = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.1, seed=26)
    a = gpu_ctx.rotation_averaging(rel, n)
    b = gpu_ctx.rotation_averaging(rel, n)
    for x, y in zip(a[:4], b[:4]):
        assert np.array_equal(x, y)
    for k in ("lm_iterations", "lm_initial_cost", "lm_final_cost", "n_valid_triplets", "init_iterations"):
        assert a[4][k] == b[4][k]


def test_invalid_inputs(gpu_ctx, r3dlib):
    rel, _, _ = make_problem(5, complete_edges(5), seed=1)
    bad = rel.copy()
    bad[0]["J"] = bad[0]["I"]
    dup = np.concatenate([rel, rel[:1]])
    dup[-1]["I"], dup[-1]["J"] = rel[0]["J"], rel[0]["I"]
    for args, code in (((bad, 5), -1), ((rel, 4), -1), ((dup, 5), -1)):
        with pytest.raises(r3dlib.R3DError) as e:
            gpu_ctx.rotation_averaging(*args)
        assert e.value.code == code
    with pytest.raises(r3dlib.R3DError) as e:
        gpu_ctx.rotation_averaging(rel, 5, method=r3dlib.ROTAVG_L1)
    assert e.value.code == -5


def test_two_devices_equal_one(r3dlib):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    n = 40
    rel, _, _ = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.1, seed=27)
    c1, c2 = r3dlib.Context((0,)), r3dlib.Context((0, 1))
    a, b = c1.rotation_averaging(rel, n), c2.rotation_averaging(rel, n)
    for x, y in zip(a[:4], b[:4]):
        assert np.array_equal(x, y)
    c1.close()
    c2.close()


def test_end_to_end_from_relative_poses(gpu_ctx, oracle):
    """relative_poses on an 8-view ring scene, then rotation_averaging: the rotations of synth.make_scene up to the gauge
    within 0.5 degrees (the relative poses carry the estimation noise of 0.5 px image noise)."""
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
    (rg, vg, _, _, S), _ = _compare(gpu_ctx, rel, n)
    assert S["success"] and vg.sum() >= 6
    assert np.degrees(gauge_error_fro(rg, np.asarray(Rs), vg) / np.sqrt(2)) < 0.5
