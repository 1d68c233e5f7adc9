"""-m gpu: the candidate keys of the integer tensor-core path (uint8 descriptors) are exact, so numpy predicts the whole
key array bit for bit: padding rows, chunk minima, float32 rounding, chunk-id packing and the order of the kept keys."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CHUNK = 8            # r3d::kChunk
NUM_KEYS = 6         # r3d::kNumKeys
KEY_STRIDE = 8       # r3d::kKeyStride
ROW_PAD = 256        # r3d::kRowPad
PAD_NORM = 1 << 28   # r3d::kPadNorm
SENTINEL = 0x7F7FFFFF


def expected_keys(db, qry):
    """Keys of every query row against database `db`, as the candidate kernel packs them."""
    n, m = len(db), len(qry)
    n_pad = (max(n, 1) + ROW_PAD - 1) // ROW_PAD * ROW_PAD
    a = np.zeros((n_pad, db.shape[1]), np.int64)
    a[:n] = db
    na = (a * a).sum(1)
    na[n:] = PAD_NORM
    q = qry.astype(np.int64)
    bracket = na[None, :] - 2 * (q @ a.T)
    cm = bracket.reshape(m, n_pad // CHUNK, CHUNK).min(2) + (q * q).sum(1)[:, None]
    nchunks = n_pad // CHUNK
    bits = max(4, int(np.ceil(np.log2(nchunks))))
    packed = cm.astype(np.float64).astype(np.float32).view(np.uint32)   # exact int -> float64, then round to nearest
    packed = (packed & np.uint32(~((1 << bits) - 1) & 0xFFFFFFFF)) | np.arange(nchunks, dtype=np.uint32)[None, :]
    out = np.full((m, KEY_STRIDE), SENTINEL, np.uint32)
    out[:, :NUM_KEYS] = np.sort(packed, 1)[:, :NUM_KEYS]   # non-negative floats order like their bit patterns
    return out


@pytest.mark.parametrize("dim", [16, 64, 128, 256])
@pytest.mark.parametrize("n", [2, 31, 33, 40, 257, 2048, 5000])
def test_integer_candidate_keys_bit_exact(gpu_ctx, dim, n):
    """n covers a partial last 32-row group, fewer than 6 real chunks and n not a multiple of the 256-row tile;
    D = 256 has two K-blocks; the query count is not a multiple of the 128-row query block."""
    rng = np.random.default_rng(1000 * dim + n)
    m = 77 + (n % 300)
    db = rng.integers(0, 256, (n, dim)).astype(np.uint8)
    qry = rng.integers(0, 256, (m, dim)).astype(np.uint8)
    k = min(n, m) // 3                 # exact duplicates: zero distances pack to denormals
    qry[:k] = db[rng.permutation(n)[:k]]
    gpu_ctx.clear_regions()
    gpu_ctx.upload_regions(0, db, rng.uniform(0, 500, (n, 2)).astype(np.float32))
    gpu_ctx.upload_regions(1, qry, rng.uniform(0, 500, (m, 2)).astype(np.float32))
    keys, eps = gpu_ctx.debug_candidate_keys(0, 1, m)
    assert eps == 0.0
    exp = expected_keys(db, qry)
    got = keys[:m]
    bad = np.nonzero((got != exp).any(1))[0]
    assert np.array_equal(got, exp), "%d of %d query rows differ, first row %d: got %s expected %s" % (
        bad.size, m, bad[0], got[bad[0]].tolist(), exp[bad[0]].tolist())
