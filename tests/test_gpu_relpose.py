"""-m gpu: r3d_relative_poses against the CPU oracle (orc_relative_poses): the same status, inlier sequence, E, errorMax
and chosen motion bit for bit; with the two-view refinement the same LM iteration / accept sequence and the final cost
within 1e-8 relative (the bars of test_gpu_ba.py)."""
import numpy as np
import pytest

from oracle import pyoracle_relpose as rpo
from regard3d_b200 import synth
from relpose_scenes import two_view

pytestmark = pytest.mark.gpu


def _Ks(widths, heights):
    return np.array([[1.1 * max(int(w), int(h)), w / 2.0, h / 2.0] for w, h in zip(widths, heights)])


def _run(ctx, oracle, r3dlib, xys, widths, heights, Ks, pairs, ofs, m, **opts):
    ctx.clear_regions()
    for v, x in enumerate(xys):
        ctx.upload_regions(v, np.zeros((len(x), 16), np.float32), x)
    put = r3dlib.Matches.from_csr(pairs, ofs, m)
    got, inl = ctx.relative_poses(put, widths, heights, Ks, **opts)
    # the map drops pairs without matches and orders by (I, J): compare in map order
    keep = [k for k in range(len(pairs)) if ofs[k + 1] > ofs[k]]
    order = sorted(keep, key=lambda k: (int(pairs[k][0]), int(pairs[k][1])))
    p2 = pairs[order]
    o2 = np.zeros(len(order) + 1, np.uint64)
    chunks = []
    for a, k in enumerate(order):
        chunks.append(m[int(ofs[k]):int(ofs[k + 1])])
        o2[a + 1] = o2[a] + len(chunks[-1])
    m2 = np.concatenate(chunks) if chunks else m[:0]
    exp, io, im = rpo.relative_poses(xys, widths, heights, Ks, p2, o2, m2, **opts)
    assert len(got) == len(exp)
    gi = inl.to_dict()
    refine = opts.get("refine", True)
    for a, (g, e) in enumerate(zip(got, exp)):
        key = (int(e["I"]), int(e["J"]))
        assert (g["I"], g["J"]) == key
        assert g["status"] == e["status"], key
        if e["status"] != rpo.RELPOSE_OK:
            assert key not in gi
            continue
        assert np.array_equal(gi[key], im[int(io[a]):int(io[a + 1])]), "pair %s: inlier sequence differs" % (key,)
        for f in ("n_inliers", "found_residual_precision", "E"):
            assert np.array_equal(g[f], e[f]), (key, f)
        if not refine:
            assert np.array_equal(g["rotation"], e["rotation"]) and np.array_equal(g["translation"], e["translation"]), key
            assert g["ba_termination"] == -1
            continue
        for f in ("ba_iterations", "ba_successful_steps", "ba_termination"):
            assert g[f] == e[f], (key, f, g[f], e[f])
        assert abs(g["ba_initial_cost"] - e["ba_initial_cost"]) <= 1e-12 * e["ba_initial_cost"], key
        assert abs(g["ba_final_cost"] - e["ba_final_cost"]) <= 1e-8 * e["ba_final_cost"], key
        # the two solves take the same steps and differ only in the rounding of the Jacobians (analytic on the device,
        # autodiff in the oracle) and of the reductions: the final cost agrees to 1e-8, the motion to far below noise
        assert np.allclose(g["rotation"], e["rotation"], atol=1e-7), key
        assert np.allclose(g["translation"], e["translation"], atol=1e-6 * max(1.0, np.abs(e["translation"]).max())), key
    return got, exp


def _scene(n, feats, seed):
    sc = synth.make_scene(n, feats, 64, "msurf", seed=seed)
    return sc, synth.exhaustive_pairs(n)


def test_clean_ring_scene(gpu_ctx, oracle, r3dlib):
    sc, pairs = _scene(5, 1500, 61)
    ofs, m = oracle.match_pairs(sc["descs"], sc["xys"], pairs, 0.8)
    Ks = _Ks(sc["widths"], sc["heights"])
    got, _ = _run(gpu_ctx, oracle, r3dlib, sc["xys"], sc["widths"], sc["heights"], Ks, pairs, ofs, m)
    assert (got["status"] == r3dlib.RELPOSE_OK).sum() >= 6
    t = gpu_ctx.relpose_timing()
    assert t["kernel_launches"] >= 4 and t["ba_iterations"] > 0
    # two calls: identical output
    got2, _ = _run(gpu_ctx, oracle, r3dlib, sc["xys"], sc["widths"], sc["heights"], Ks, pairs, ofs, m)
    for f in r3dlib.relpose_dtype.names:   # field by field: the struct's padding bytes carry no value
        assert np.array_equal(got[f], got2[f]), f
    # refine = 0: the unrefined motion, bit for bit
    _run(gpu_ctx, oracle, r3dlib, sc["xys"], sc["widths"], sc["heights"], Ks, pairs, ofs, m, refine=False)


def test_random_matches_tiny_pairs_and_missing_intrinsics(gpu_ctx, oracle, r3dlib):
    sc, pairs = _scene(4, 1500, 62)
    ofs, m = oracle.match_pairs(sc["descs"], sc["xys"], pairs, 0.8)
    rng = np.random.default_rng(3)
    m2 = m.copy()
    s1 = slice(int(ofs[1]), int(ofs[2]))
    m2["j"][s1] = rng.permutation(1500)[: int(ofs[2] - ofs[1])]     # pair 1: random matches
    keep = np.ones(len(m2), bool)
    keep[int(ofs[2]) + 9:int(ofs[3])] = False                       # pair (0, 3): 9 matches
    keep[int(ofs[3]) + 5:int(ofs[4])] = False                       # pair (1, 2): 5 matches
    new_ofs = np.zeros_like(ofs)
    for k in range(len(pairs)):
        new_ofs[k + 1] = new_ofs[k] + keep[int(ofs[k]):int(ofs[k + 1])].sum()
    m2 = m2[keep]
    Ks = _Ks(sc["widths"], sc["heights"])
    Ks[3, 0] = 0.0                                                  # view 3: no pinhole intrinsic
    got, _ = _run(gpu_ctx, oracle, r3dlib, sc["xys"], sc["widths"], sc["heights"], Ks, pairs, new_ofs, m2)
    st = {(int(g["I"]), int(g["J"])): int(g["status"]) for g in got}
    assert st[(0, 2)] == r3dlib.RELPOSE_NO_MODEL and st[(1, 2)] == r3dlib.RELPOSE_TOO_FEW
    assert st[(0, 3)] == r3dlib.RELPOSE_NO_INTRINSIC and st[(1, 3)] == r3dlib.RELPOSE_NO_INTRINSIC
    assert st[(0, 1)] == r3dlib.RELPOSE_OK


def _pair_views(specs):
    """views / pairs / matches from two_view() pairs laid out as consecutive view pairs (2k, 2k + 1)."""
    xys, pairs, ofs, chunks = [], [], [0], []
    for k, (xI, xJ) in enumerate(specs):
        xys += [xI, xJ]
        pairs.append((2 * k, 2 * k + 1))
        n = len(xI)
        chunks.append(np.array(list(zip(range(n), range(n))), dtype=[("i", np.uint32), ("j", np.uint32)]))
        ofs.append(ofs[-1] + n)
    return xys, np.array(pairs, np.uint32), np.array(ofs, np.uint64), np.concatenate(chunks)


def _mixed(outlier_frac, rotation_pair):
    specs = []
    for k, n in enumerate((6, 12, 40, 300, 2500)):
        xI, xJ, _, _, _ = two_view(n, seed=100 + k, outlier_frac=outlier_frac)
        specs.append((xI, xJ))
    if rotation_pair:
        xI, xJ, _, _, _ = two_view(800, seed=7, baseline=(1e-4, 0.0, 0.0), rot=(0.0, 0.2, 0.0))  # near-pure rotation
        specs.append((xI, xJ))
    # more than 16384 matches in one pair: the huge AC-RANSAC class and the largest BA scratch slot
    xI, xJ, _, _, _ = two_view(17000, seed=8, outlier_frac=1.5 * outlier_frac)
    specs.append((xI, xJ))
    return _pair_views(specs)


def test_mixed_batch_rotation_pair_and_huge_pair(gpu_ctx, oracle, r3dlib):
    # gross outliers, a near-pure rotation: AC-RANSAC, E and the chosen motion bit for bit
    xys, pairs, ofs, m = _mixed(0.2, True)
    n = len(xys)
    widths, heights = np.full(n, 1920, np.uint32), np.full(n, 1080, np.uint32)
    got, _ = _run(gpu_ctx, oracle, r3dlib, xys, widths, heights, _Ks(widths, heights), pairs, ofs, m, refine=False)
    assert got["status"][0] == r3dlib.RELPOSE_NO_MODEL and got["status"][-1] == r3dlib.RELPOSE_OK  # 6 matches: < 13 inliers
    assert got["n_inliers"][-1] > 10000
    # the refinement on matches without gross outliers (what matches.e.txt holds).  A bad match gives a DLT point that
    # the Huber loss lets slide for hundreds of LM iterations; over such runs the rounding of the Jacobians (analytic
    # here, autodiff in the oracle) can shift an accept decision, so the step-for-step bar applies to converging solves
    xys, pairs, ofs, m = _mixed(0.0, False)
    got, _ = _run(gpu_ctx, oracle, r3dlib, xys, widths[:len(xys)], heights[:len(xys)], _Ks(widths, heights)[:len(xys)], pairs,
                  ofs, m)
    assert (got["status"] == r3dlib.RELPOSE_OK).sum() == len(got) - 2 and got["ba_iterations"].max() < 50


def test_cross_check_against_bundle_adjust(gpu_ctx, oracle, r3dlib):
    """One pair's refinement against r3d_bundle_adjust on the same two-camera problem."""
    xI, xJ, _, _, K = two_view(500, seed=11)
    xys, pairs, ofs, m = _pair_views([(xI, xJ)])
    widths, heights = np.full(2, 1920, np.uint32), np.full(2, 1080, np.uint32)
    Ks = _Ks(widths, heights)
    r0, _ = _run(gpu_ctx, oracle, r3dlib, xys, widths, heights, Ks, pairs, ofs, m, refine=False)
    r1, _ = _run(gpu_ctx, oracle, r3dlib, xys, widths, heights, Ks, pairs, ofs, m)
    R, t = r0[0]["rotation"], r0[0]["translation"]
    c = np.clip((np.trace(R) - 1) / 2, -1, 1)
    th = np.arccos(c)
    aa = th / (2 * np.sin(th)) * np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    Km = np.array([[K[0], 0, K[1]], [0, K[0], K[2]], [0, 0, 1.0]])
    P1, P2 = Km @ np.c_[np.eye(3), np.zeros(3)], Km @ np.c_[R, t]
    X = []
    for a, b in zip(xI.astype(np.float64), xJ.astype(np.float64)):
        A = np.stack([a[0] * P1[2] - P1[0], a[1] * P1[2] - P1[1], b[0] * P2[2] - P2[0], b[1] * P2[2] - P2[1]])
        X.append(np.linalg.lstsq(A[:, :3], -A[:, 3], rcond=None)[0])
    n = len(xI)
    p = {"poses": np.array([np.zeros(6), np.r_[aa, t]]), "intrinsics": np.array([[K[0], K[1], K[2], 0, 0, 0]] * 2),
         "points": np.array(X), "obs_cam": np.tile(np.array([0, 1], np.uint32), n),
         "obs_pt": np.repeat(np.arange(n, dtype=np.uint32), 2), "cam_intr": np.array([0, 1], np.uint32),
         "obs_xy": np.stack([xI.astype(np.float64), xJ.astype(np.float64)], 1).reshape(-1, 2)}
    p = {k: np.ascontiguousarray(v) for k, v in p.items()}
    s, _ = gpu_ctx.bundle_adjust(p, refine_intrinsics=0)
    # the starting points differ in the last bits (numpy's DLT): the same minimum, not the same steps
    assert abs(s["final_cost"] - r1[0]["ba_final_cost"]) < 1e-6 * s["final_cost"]


def test_two_devices_equal_one(r3dlib, oracle):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    sc, pairs = _scene(5, 1500, 63)
    ofs, m = oracle.match_pairs(sc["descs"], sc["xys"], pairs, 0.8)
    Ks = _Ks(sc["widths"], sc["heights"])
    outs = []
    for devs in ((0,), (0, 1)):
        ctx = r3dlib.Context(devs)
        for v, x in enumerate(sc["xys"]):
            ctx.upload_regions(v, sc["descs"][v], x)
        got, inl = ctx.relative_poses(r3dlib.Matches.from_csr(pairs, ofs, m), sc["widths"], sc["heights"], Ks)
        outs.append((got.tobytes(), {k: v.tobytes() for k, v in inl.to_dict().items()}))
        ctx.close()
    assert outs[0] == outs[1]
