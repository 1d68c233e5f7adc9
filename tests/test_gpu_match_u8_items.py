"""-m gpu: the integer candidate path works on 256-query work items (two 128-row query boxes, four consumer
warpgroups); the fp16 path keeps 128-query items.  Query counts around the 256-row block, where the second box is
empty or partly past the view, against a numpy restatement of the keys and against the CPU oracle."""
import numpy as np
import pytest

from conftest import dict_sets, match_sets
from regard3d_b200 import synth

pytestmark = pytest.mark.gpu

CHUNK = 8            # r3d::kChunk
NUM_KEYS = 6         # r3d::kNumKeys
KEY_STRIDE = 8       # r3d::kKeyStride
ROW_PAD = 256        # r3d::kRowPad
PAD_NORM = 1 << 28   # r3d::kPadNorm
SENTINEL = 0x7F7FFFFF


def expected_keys(db, qry):
    """Keys of every query row against database `db`, as the candidate kernel packs them: the chunk minima of the
    exact squared distances, rounded to float32, chunk id in the low bits, the NUM_KEYS smallest in order."""
    n, m = len(db), len(qry)
    n_pad = (max(n, 1) + ROW_PAD - 1) // ROW_PAD * ROW_PAD
    a = np.zeros((n_pad, db.shape[1]), np.int64)
    a[:n] = db
    na = (a * a).sum(1)
    na[n:] = PAD_NORM
    q = qry.astype(np.int64)
    cm = (na[None, :] - 2 * (q @ a.T)).reshape(m, n_pad // CHUNK, CHUNK).min(2) + (q * q).sum(1)[:, None]
    nchunks = n_pad // CHUNK
    bits = max(4, int(np.ceil(np.log2(nchunks))))
    packed = cm.astype(np.float64).astype(np.float32).view(np.uint32)
    packed = (packed & np.uint32(~((1 << bits) - 1) & 0xFFFFFFFF)) | np.arange(nchunks, dtype=np.uint32)[None, :]
    out = np.full((m, KEY_STRIDE), SENTINEL, np.uint32)
    out[:, :NUM_KEYS] = np.sort(packed, 1)[:, :NUM_KEYS]
    return out


def _check_keys(gpu_ctx, n, m, dim, seed):
    rng = np.random.default_rng(seed)
    db = rng.integers(0, 256, (n, dim)).astype(np.uint8)
    qry = rng.integers(0, 256, (m, dim)).astype(np.uint8)
    k = min(n, m) // 3
    qry[:k] = db[rng.permutation(n)[:k]]
    gpu_ctx.clear_regions()
    gpu_ctx.upload_regions(0, db, rng.uniform(0, 500, (n, 2)).astype(np.float32))
    gpu_ctx.upload_regions(1, qry, rng.uniform(0, 500, (m, 2)).astype(np.float32))
    keys, eps = gpu_ctx.debug_candidate_keys(0, 1, m)
    assert eps == 0.0
    exp = expected_keys(db, qry)
    got = keys[:m]
    bad = np.nonzero((got != exp).any(1))[0]
    assert bad.size == 0, "%d of %d query rows differ, first row %d: got %s expected %s" % (
        bad.size, m, bad[0], got[bad[0]].tolist(), exp[bad[0]].tolist())


@pytest.mark.parametrize("dim", [64, 128, 256])
@pytest.mark.parametrize("m", [1, 129, 255, 256, 257, 300])
def test_keys_around_the_256_row_block(gpu_ctx, dim, m):
    """m <= 128: the second query box of the block lies wholly past the view; 129..255: partly; 257 and 300: a second
    block.  D = 256 has two K-blocks and a single query buffer."""
    _check_keys(gpu_ctx, 700, m, dim, seed=31 * dim + m)


@pytest.mark.parametrize("dim", [64, 128, 256])
def test_keys_several_blocks_and_tiles(gpu_ctx, dim):
    _check_keys(gpu_ctx, 5000, 2048, dim, seed=dim)


def _upload(ctx, descs, xys, first=0):
    for v, (d, x) in enumerate(zip(descs, xys)):
        ctx.upload_regions(first + v, d, x)


def _ragged_views(rng, sizes, dim):
    descs = [rng.integers(0, 256, (n, dim)).astype(np.uint8) for n in sizes]
    src = descs[int(np.argmax(sizes))]
    for v in range(len(sizes)):            # near-duplicates of the largest view's rows so that ratio tests pass
        k = min(sizes[v], 300)
        noise = rng.integers(-3, 4, (k, dim))
        descs[v][:k] = np.clip(src[rng.permutation(len(src))[:k]].astype(np.int64) + noise, 0, 255).astype(np.uint8)
    xys = [rng.uniform(0, 500, (n, 2)).astype(np.float32) for n in sizes]
    return descs, xys


def test_u8_ragged_views_match_oracle(gpu_ctx, oracle, r3dlib):
    rng = np.random.default_rng(5)
    descs, xys = _ragged_views(rng, [0, 1, 257, 1000, 4100], 128)
    pairs = synth.exhaustive_pairs(len(descs))
    gpu_ctx.clear_regions()
    _upload(gpu_ctx, descs, xys)
    ofs, m = oracle.match_pairs(descs, xys, pairs, 0.9)
    exp = match_sets(ofs, m, pairs)
    assert sum(len(s) for s in exp.values()) > 100
    for flags in (r3dlib.MATCH_DEFAULT, r3dlib.MATCH_EXACT_SCAN):
        got = dict_sets(gpu_ctx.match_pairs(pairs, 0.9, flags).to_dict())
        assert got == exp, "flags=%d" % flags


@pytest.mark.parametrize("other", ["u8-72", "f32-128"])
def test_integer_and_fp16_items_in_one_context(gpu_ctx, oracle, r3dlib, other):
    """Views of the integer path (u8 D = 128, 256-query items) and of the fp16 path (u8 D = 72 or float32, 128-query
    items) uploaded side by side and matched in separate calls."""
    rng = np.random.default_rng(11)
    u8_descs, u8_xys = _ragged_views(rng, [300, 700, 1200], 128)
    sc = synth.make_scene(3, 600, 72 if other == "u8-72" else 128, "sift", seed=12, as_u8=(other == "u8-72"))
    gpu_ctx.clear_regions()
    _upload(gpu_ctx, u8_descs, u8_xys)
    _upload(gpu_ctx, sc["descs"], sc["xys"], first=3)
    pairs = synth.exhaustive_pairs(3)
    for descs, xys, first in ((u8_descs, u8_xys, 0), (sc["descs"], sc["xys"], 3)):
        ofs, m = oracle.match_pairs(descs, xys, pairs, 0.8)
        exp = match_sets(ofs, m, pairs)
        assert sum(len(s) for s in exp.values()) > 50
        for flags in (r3dlib.MATCH_DEFAULT, r3dlib.MATCH_EXACT_SCAN):
            got = dict_sets(gpu_ctx.match_pairs(pairs + first, 0.8, flags).to_dict())
            got = {(I - first, J - first): s for (I, J), s in got.items()}
            assert got == exp, "views %d.., flags=%d" % (first, flags)
