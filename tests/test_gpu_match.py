"""-m gpu: the CUDA matching path through the C ABI vs the CPU oracle -- bit-exact (i,j) sets."""
import numpy as np
import pytest

import fp16_keys_ref as ref
from conftest import dict_sets, match_sets
from regard3d_b200 import synth

pytestmark = pytest.mark.gpu


def _upload(ctx, sc):
    ctx.clear_regions()
    for v, (d, x) in enumerate(zip(sc["descs"], sc["xys"])):
        ctx.upload_regions(v, d, x)


@pytest.mark.parametrize("kind,dim,n,as_u8", [
    ("msurf", 64, 1500, False), ("liop", 144, 1500, False), ("sift", 128, 1500, False),
    ("sift", 128, 1500, True), ("msurf", 61, 700, False), ("msurf", 32, 300, False),
])
def test_match_pairs_equals_oracle(gpu_ctx, oracle, r3dlib, kind, dim, n, as_u8):
    sc = synth.make_scene(4, n, dim, kind, seed=7, as_u8=as_u8)
    pairs = synth.exhaustive_pairs(4)
    _upload(gpu_ctx, sc)
    ofs, m = oracle.match_pairs(sc["descs"], sc["xys"], pairs, 0.6)
    exp = match_sets(ofs, m, pairs)
    for flags in (r3dlib.MATCH_DEFAULT, r3dlib.MATCH_EXACT_SCAN):
        got = dict_sets(gpu_ctx.match_pairs(pairs, 0.6, flags).to_dict())
        assert got == exp, "flags=%d" % flags
    t = gpu_ctx.match_timing()
    assert t["kernel_launches"] >= 2


def test_order_of_output_is_the_references_set_order(gpu_ctx, oracle):
    sc = synth.make_scene(2, 2000, 64, "msurf", seed=9)
    pairs = synth.exhaustive_pairs(2)
    _upload(gpu_ctx, sc)
    ofs, m = oracle.match_pairs(sc["descs"], sc["xys"], pairs, 0.7)
    I, J, g = gpu_ctx.match_pairs(pairs, 0.7).pair(0)
    assert (I, J) == (0, 1)
    assert np.array_equal(g, m)        # same sequence, not only the same set (std::set iteration order)


def test_ragged_and_degenerate_views(gpu_ctx, oracle, r3dlib):
    rng = np.random.default_rng(3)
    sizes = [0, 1, 2, 5, 257, 1000]
    descs = [rng.standard_normal((n, 48)).astype(np.float32) for n in sizes]
    descs = [d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-9) if len(d) else d for d in descs]
    xys = [rng.uniform(0, 500, (n, 2)).astype(np.float32) for n in sizes]
    pairs = synth.exhaustive_pairs(len(sizes))
    gpu_ctx.clear_regions()
    for v in range(len(sizes)):
        gpu_ctx.upload_regions(v, descs[v], xys[v])
    ofs, m = oracle.match_pairs(descs, xys, pairs, 0.9)
    exp = match_sets(ofs, m, pairs)
    for flags in (r3dlib.MATCH_DEFAULT, r3dlib.MATCH_EXACT_SCAN):
        got = dict_sets(gpu_ctx.match_pairs(pairs, 0.9, flags).to_dict())
        assert got == exp


def test_duplicate_descriptors_and_ties(gpu_ctx, oracle):
    # exact duplicates in the database (ties between best and second) and duplicated coordinates
    sc = synth.make_scene(2, 1200, 64, "msurf", seed=12)
    d0 = sc["descs"][0].copy()
    d0[100:200] = d0[0:100]                      # duplicate rows -> d1 == d2 for their matches
    x1 = sc["xys"][1].copy()
    x1[1::2] = x1[0::2]                          # pairs of features share coordinates
    descs = [d0, sc["descs"][1]]
    xys = [sc["xys"][0], x1]
    pairs = synth.exhaustive_pairs(2)
    gpu_ctx.clear_regions()
    for v in range(2):
        gpu_ctx.upload_regions(v, descs[v], xys[v])
    ofs, m = oracle.match_pairs(descs, xys, pairs, 0.8)
    got = dict_sets(gpu_ctx.match_pairs(pairs, 0.8).to_dict())
    assert got == match_sets(ofs, m, pairs)


def test_search_neighbours_bit_exact(gpu_ctx, oracle):
    sc = synth.make_scene(2, 3000, 144, "liop", seed=13)
    _upload(gpu_ctx, sc)
    idx, dist = gpu_ctx.search_neighbours(0, 1, 3000)
    oi, od = oracle.search_neighbours(sc["descs"][0], sc["descs"][1])
    assert np.array_equal(idx, oi)
    assert np.array_equal(dist.view(np.uint32), od.view(np.uint32))


def test_candidate_error_bound_holds(gpu_ctx):
    """The certification relies on |candidate value - real distance| <= eps_abs + 2^(b-23) |value|: checked term by term
    against the float64 reference (fp16_keys_ref.check_pair) on LIOP-144, 2048 x 2048.  The other shapes and data kinds
    are in tests/test_gpu_match_fp16_bound.py."""
    sc = synth.make_scene(2, 2048, 144, "liop", seed=14)
    _upload(gpu_ctx, sc)
    ref.check_pair(gpu_ctx, 0, 1, sc["descs"][0], sc["descs"][1], "synthetic LIOP-144 2048x2048")


def test_full_size_properties_c2_slice(gpu_ctx, r3dlib):
    """BASELINE C2 feature counts (10k x 10k, D=144) on a 4-image slice: tensor-core path ==
    exact-scan path (size-independent property: both are the same function), symmetry of counts."""
    sc = synth.make_scene(4, 10000, 144, "liop", seed=15)
    pairs = synth.exhaustive_pairs(4)
    _upload(gpu_ctx, sc)
    a = dict_sets(gpu_ctx.match_pairs(pairs, 0.6).to_dict())
    t = gpu_ctx.match_timing()
    b = dict_sets(gpu_ctx.match_pairs(pairs, 0.6, r3dlib.MATCH_EXACT_SCAN).to_dict())
    assert a == b
    assert t["fallback_queries"] < 0.05 * t["queries"]
    truth = sc["truth"]
    for (I, J), s in a.items():
        ok = sum(1 for (i, j) in s if truth[I][i] == truth[J][j] and truth[I][i] >= 0)
        assert ok >= 0.98 * len(s)


@pytest.mark.parametrize("case", ["dim256_f32", "dim300_u8", "huge_values", "mixed_range"])
def test_descriptors_outside_the_fp16_operand_range_take_the_exact_scan(gpu_ctx, oracle, r3dlib, case):
    """Round 1 returned R3D_ERR_UNSUPPORTED for descriptor dimensions > 240 and values beyond the fp16 operands;
    such views now keep their exact descriptors only and their pairs are matched by the exact CUDA-core scan."""
    rng = np.random.default_rng(17)
    n, nv = 600, 3
    if case == "dim256_f32":
        descs = [rng.standard_normal((n, 256)).astype(np.float32) for _ in range(nv)]
    elif case == "dim300_u8":
        descs = [rng.integers(0, 256, (n, 300)).astype(np.uint8) for _ in range(nv)]
    elif case == "huge_values":
        descs = [(rng.standard_normal((n, 64)) * 1e5).astype(np.float32) for _ in range(nv)]
    else:                                                    # one view out of range, the others on the tensor path
        descs = [rng.standard_normal((n, 64)).astype(np.float32) for _ in range(nv)]
        descs[1] = (descs[1] * 5e4).astype(np.float32)
    for v in range(1, nv):                                   # plant true correspondences so the ratio test passes
        descs[v][:200] = descs[0][:200]
        if descs[v].dtype != np.uint8:
            descs[v][:200] += (0.01 * np.abs(descs[0][:200]).mean() * rng.standard_normal((200, descs[v].shape[1]))).astype(np.float32)
    if case == "mixed_range":
        descs[1] = descs[1].astype(np.float32)
    xys = [rng.uniform(0, 900, (n, 2)).astype(np.float32) for _ in range(nv)]
    pairs = synth.exhaustive_pairs(nv)
    gpu_ctx.clear_regions()
    for v in range(nv):
        gpu_ctx.upload_regions(v, descs[v], xys[v])
    ofs, m = oracle.match_pairs(descs, xys, pairs, 0.8)
    got = dict_sets(gpu_ctx.match_pairs(pairs, 0.8).to_dict())
    assert got == match_sets(ofs, m, pairs) and sum(len(s) for s in got.values()) > 100
    gpu_ctx.clear_regions()


def test_mutual_nn_flag(gpu_ctx, oracle, r3dlib):
    """R3D_MATCH_MUTUAL_NN (off by default; not reference behaviour): forward ratio matches whose I-feature also has the
    J-feature as ITS nearest neighbour -- checked against the oracle's SearchNeighbours in both directions."""
    sc = synth.make_scene(3, 1200, 64, "msurf", seed=21)
    pairs = synth.exhaustive_pairs(3)
    _upload(gpu_ctx, sc)
    plain = gpu_ctx.match_pairs(pairs, 0.7).to_dict()
    mutual = gpu_ctx.match_pairs(pairs, 0.7, r3dlib.MATCH_MUTUAL_NN).to_dict()
    n_plain = n_mut = 0
    for (I, J), m in plain.items():
        idx, _ = oracle.search_neighbours(sc["descs"][J], sc["descs"][I])          # for every i of I: its 2-NN in J
        want = [(int(i), int(j)) for i, j in zip(m["i"], m["j"]) if idx[i, 0] == j]
        got = mutual.get((I, J))
        got = [] if got is None else list(zip(got["i"].tolist(), got["j"].tolist()))
        assert got == want, (I, J)
        n_plain += len(m); n_mut += len(want)
    assert 0 < n_mut <= n_plain
