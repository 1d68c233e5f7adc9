"""-m gpu: r3d_translation_averaging against the CPU oracle (orc_translation_averaging), both methods: view_kept,
edge_kept, success, the counts, the LM iterations, successful steps and termination identical; the initial cost within
1e-9 and the final cost within 1e-8 relative; centres and translations within 1e-8 of the scene's scale.  And the chain
relative poses -> rotations -> translations -> structure -> bundle adjustment on a synthetic ring."""
import numpy as np
import pytest

from oracle import pyoracle_transavg as pto
from regard3d_b200 import synth
from relpose_scenes import ring_truth
from transavg_scenes import aligned_error, banded_ring, complete_edges, make_problem

pytestmark = pytest.mark.gpu

METHODS = [pto.TRANSAVG_L2_CHORDAL, pto.TRANSAVG_SOFTL1]


def _compare(gpu_ctx, rel, Rs, rk, n, method, **kw):
    got = gpu_ctx.translation_averaging(rel, Rs, rk, n, method=method, **kw)
    exp = pto.translation_averaging(rel, Rs, rk, n, method=method, **kw)
    Cg, Tg, vg, eg, Sg = got
    Co, To, vo, eo, So = exp
    for k in ("success", "n_edges", "n_kept_edges", "n_kept_views", "lm_iterations", "lm_successful_steps", "lm_termination"):
        assert Sg[k] == So[k], (k, Sg[k], So[k])
    assert np.array_equal(vg, vo) and np.array_equal(eg, eo)
    if not So["success"]:
        assert not Cg.any() and not Tg.any()
        return got, exp
    assert abs(Sg["lm_initial_cost"] - So["lm_initial_cost"]) <= 1e-9 * max(So["lm_initial_cost"], 1e-300)
    assert abs(Sg["lm_final_cost"] - So["lm_final_cost"]) <= 1e-8 * max(So["lm_final_cost"], 1e-300)
    scale = max(np.abs(Co[vo]).max(), np.abs(To[vo]).max(), 1e-300)
    assert np.abs(Cg - Co).max() <= 1e-8 * scale and np.abs(Tg - To).max() <= 1e-8 * scale
    return got, exp


@pytest.mark.parametrize("method", METHODS)
def test_complete_graph(gpu_ctx, method):
    n = 60
    rel, Rs, Cs, _ = make_problem(n, complete_edges(n), noise_deg=0.5, seed=31)
    (C, _, vk, _, S), _ = _compare(gpu_ctx, rel, Rs, np.ones(n, bool), n, method)
    assert S["success"] and S["n_kept_views"] == n and S["lm_iterations"] > 0
    assert aligned_error(C, Cs, vk) < 0.01
    assert S["ms_solve"] > 0 and S["ms_device_total"] >= S["ms_solve"]


@pytest.mark.parametrize("method", METHODS)
def test_banded_ring(gpu_ctx, method):
    n = 200
    rel, Rs, Cs, _ = make_problem(n, banded_ring(n, 3), noise_deg=0.5, seed=32)
    (C, _, vk, _, S), _ = _compare(gpu_ctx, rel, Rs, np.ones(n, bool), n, method)
    assert S["n_kept_views"] == n


@pytest.mark.parametrize("method", METHODS)
def test_bridge_pendant_unusable_records(gpu_ctx, method):
    # views 0..9 dense, 10..15 dense, bridge (9, 10), pendant 16 on 3; 17..19 without edges; a record that is not OK, one
    # with edge_use = 0 and a view that rotation averaging did not keep
    e = [(i, j) for i in range(10) for j in range(i + 1, 10)] + [(i, j) for i in range(10, 16) for j in range(i + 1, 16)]
    e += [(9, 10), (3, 16)]
    rel, Rs, _, _ = make_problem(20, e, noise_deg=0.3, seed=33)
    rel["status"][1] = pto.RELPOSE_NO_MODEL
    use = np.ones(len(rel), bool)
    use[2] = False
    rk = np.ones(20, bool)
    rk[4] = False
    (C, T, vk, ek, S), _ = _compare(gpu_ctx, rel, Rs, rk, 20, method, edge_use=use)
    assert set(np.nonzero(vk)[0].tolist()) == set(range(10)) - {4}
    assert not C[~vk].any() and not T[~vk].any() and not ek[1] and not ek[2]


def test_softl1_active_bounds(gpu_ctx):
    """Scale factors spread over [0.3, 3]: at the optimum part of the scales sit on the bound s = 1."""
    n = 40
    rel, Rs, _, _ = make_problem(n, complete_edges(n), noise_deg=1.0, seed=34, scale_range=(0.3, 3.0))
    (C, T, vk, _, S), _ = _compare(gpu_ctx, rel, Rs, np.ones(n, bool), n, pto.TRANSAVG_SOFTL1)
    t = rel["translation"] / np.linalg.norm(rel["translation"], axis=1, keepdims=True)
    I, J = rel["I"].astype(int), rel["J"].astype(int)
    q = T[J] - np.einsum("eab,ecb,ec->ea", Rs[J], Rs[I], T[I])
    assert ((q * t).sum(1) < 1.0).any()                      # the bound is active for some edges


@pytest.mark.parametrize("method", METHODS)
def test_repeated_calls_are_bit_identical(gpu_ctx, method):
    n = 50
    rel, Rs, _, _ = make_problem(n, complete_edges(n), noise_deg=0.5, outlier_frac=0.05, seed=35)
    a = gpu_ctx.translation_averaging(rel, Rs, np.ones(n, bool), n, method=method)
    b = gpu_ctx.translation_averaging(rel, Rs, np.ones(n, bool), n, method=method)
    for x, y in zip(a[:4], b[:4]):
        assert np.array_equal(x, y)
    for k in ("lm_iterations", "lm_initial_cost", "lm_final_cost", "lm_termination"):
        assert a[4][k] == b[4][k]


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
    for r, n in ((bad, 5), (rel, 4), (dup, 5), (zero, 5), (inf, 5)):
        with pytest.raises(r3dlib.R3DError) as e:
            gpu_ctx.translation_averaging(r, Rs, rk, n)
        assert e.value.code == -1
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
    for method in METHODS:
        a = c1.translation_averaging(rel, Rs, np.ones(n, bool), n, method=method)
        b = c2.translation_averaging(rel, Rs, np.ones(n, bool), n, method=method)
        for x, y in zip(a[:4], b[:4]):
            assert np.array_equal(x, y)
    c1.close()
    c2.close()


@pytest.mark.parametrize("method", METHODS)
def test_end_to_end_relative_poses_to_bundle_adjustment(gpu_ctx, r3dlib, method):
    """match_pairs -> relative_poses -> rotation_averaging -> translation_averaging -> SfmData with these poses ->
    tracks of the AC-RANSAC inliers -> structure_from_tracks -> remove_outliers -> sfm_bundle_adjust on an 8-view ring:
    centres of synth.make_scene after a similarity alignment, and the reprojection RMS after BA."""
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
    (C, T, vk, _, S), _ = _compare(gpu_ctx, rel, Rg, rk, n, method, edge_use=ek_rot)
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
    print("end-to-end method %d: centre error %.3g of the diameter, %d landmarks, RMS %.3f px" % (method, err, len(lms), rms))
    # bars from an H100 run (centre error 2.1e-4 / 2.5e-4 of the diameter, RMS 0.600 px) with margin
    assert len(lms) > 1000
    assert err < 2e-3
    assert rms < 0.8
