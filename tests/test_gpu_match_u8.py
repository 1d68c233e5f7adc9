"""-m gpu: uint8 descriptors on the integer tensor-core path (u8 x u8 -> s32 wgmma, exact keys) and the u8 shapes
that keep the fp16 operands, against the CPU oracle."""
import numpy as np
import pytest

from conftest import dict_sets, match_sets
from regard3d_b200 import synth

pytestmark = pytest.mark.gpu


def _upload(ctx, descs, xys):
    ctx.clear_regions()
    for v, (d, x) in enumerate(zip(descs, xys)):
        ctx.upload_regions(v, d, x)


def test_integer_candidate_keys_are_exact(gpu_ctx):
    """u8 SIFT D = 128: eps_abs = 0, and every key is the packed exact chunk minimum (only the chunk-id bits differ)."""
    sc = synth.make_scene(2, 2048, 128, "sift", seed=14, as_u8=True)
    _upload(gpu_ctx, sc["descs"], sc["xys"])
    keys, eps = gpu_ctx.debug_candidate_keys(0, 1, 2048)
    assert eps == 0.0
    A = sc["descs"][0].astype(np.int64)
    B = sc["descs"][1].astype(np.int64)
    D = (B * B).sum(1)[:, None] + (A * A).sum(1)[None, :] - 2 * B @ A.T
    CH = 8                                     # r3d::kChunk
    cm = D.reshape(2048, 2048 // CH, CH).min(2).astype(np.float64)
    bits = 8                                   # 2048 rows / 8 = 256 chunks
    kv = keys[:2048, :6].view(np.float32).astype(np.float64)
    kc = (keys[:2048, :6] & ((1 << bits) - 1)).astype(np.int64)
    pack = 2.0 ** (bits - 23)
    true_at = np.take_along_axis(cm, kc, 1)
    assert (np.abs(kv - true_at) <= np.abs(kv) * pack + 1e-37).all()   # 1e-37: a zero distance packs to a denormal
    srt = np.sort(cm, 1)[:, :6]
    assert (np.abs(kv - srt) <= 2 * np.abs(srt) * pack + 1e-37).all()
    assert (np.diff(kv, axis=1) >= 0).all()


@pytest.mark.parametrize("dim,n", [(64, 1100), (72, 700), (256, 600)])
def test_u8_match_pairs_equals_oracle(gpu_ctx, oracle, r3dlib, dim, n):
    """D = 64 and 256 take the integer path, D = 72 (not a multiple of 16) the fp16 operands; n is not a multiple of
    the 256-row tile."""
    sc = synth.make_scene(4, n, dim, "sift", seed=7, as_u8=True)
    pairs = synth.exhaustive_pairs(4)
    _upload(gpu_ctx, sc["descs"], sc["xys"])
    ofs, m = oracle.match_pairs(sc["descs"], sc["xys"], pairs, 0.6)
    exp = match_sets(ofs, m, pairs)
    assert sum(len(s) for s in exp.values()) > 100
    for flags in (r3dlib.MATCH_DEFAULT, r3dlib.MATCH_EXACT_SCAN):
        got = dict_sets(gpu_ctx.match_pairs(pairs, 0.6, flags).to_dict())
        assert got == exp, "flags=%d" % flags


def test_u8_ragged_and_degenerate_views(gpu_ctx, oracle, r3dlib):
    rng = np.random.default_rng(3)
    sizes = [0, 1, 2, 5, 257, 1000]
    descs = [rng.integers(0, 256, (n, 48)).astype(np.uint8) for n in sizes]
    for v in range(1, len(sizes)):            # near-duplicates of view 5's rows so that some ratio tests pass
        k = min(sizes[v], 200)
        noise = rng.integers(-3, 4, (k, 48))
        descs[v][:k] = np.clip(descs[5][:k].astype(np.int64) + noise, 0, 255).astype(np.uint8)
    xys = [rng.uniform(0, 500, (n, 2)).astype(np.float32) for n in sizes]
    pairs = synth.exhaustive_pairs(len(sizes))
    _upload(gpu_ctx, descs, xys)
    ofs, m = oracle.match_pairs(descs, xys, pairs, 0.9)
    exp = match_sets(ofs, m, pairs)
    for flags in (r3dlib.MATCH_DEFAULT, r3dlib.MATCH_EXACT_SCAN):
        got = dict_sets(gpu_ctx.match_pairs(pairs, 0.9, flags).to_dict())
        assert got == exp
