"""-m gpu: tie-heavy inputs for the integer candidate keys.  Many chunks reach the same (or an adjacent) packed key, so
the kernel's integer pre-filter meets its set bound exactly and only the chunk bits decide which keys are kept.  numpy
predicts the whole key array bit for bit (test_gpu_candidate_keys_u8.expected_keys)."""
import numpy as np
import pytest

from test_gpu_candidate_keys_u8 import expected_keys

pytestmark = pytest.mark.gpu


def tie_case(kind, dim, n, m, rng):
    if kind == "constant":        # every real chunk at the same distance: the lowest chunk ids win
        db = np.full((n, dim), 97, np.uint8)
        qry = np.full((m, dim), 101, np.uint8)
        qry[m // 2:] = 97         # zero distances: denormal keys
    elif kind == "duplicated":    # a few distinct rows, each repeated over many chunks
        base = rng.integers(0, 256, (5, dim)).astype(np.uint8)
        db = base[rng.integers(0, len(base), n)]
        qry = base[rng.integers(0, len(base), m)].copy()
        qry[::3, 0] ^= 1          # ... and rows one unit away
    elif kind == "ramp":          # integer distances 1 apart, across the packing's rounding and truncation steps
        db = np.full((n, dim), 128, np.uint8)
        db[:, 0] = (np.arange(n) * 7) % 256
        db[:, 1] = (np.arange(n) // 256) % 256
        qry = np.full((m, dim), 128, np.uint8)
        qry[:, 0] = rng.integers(0, 256, m)
        qry[:, 2] = rng.integers(0, 256, m)
    else:                         # zero rows beside padding rows (n not a multiple of the 256-row tile)
        db = np.zeros((n, dim), np.uint8)
        db[n // 2:] = rng.integers(0, 2, (n - n // 2, dim))
        qry = np.zeros((m, dim), np.uint8)
        qry[1::2] = 255
    return db, qry


KINDS = ["constant", "duplicated", "ramp", "zero_and_pad"]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("dim,n", [(128, 5000), (128, 20000), (64, 3001), (256, 2600)])
def test_integer_candidate_keys_ties_bit_exact(gpu_ctx, kind, dim, n):
    rng = np.random.default_rng([KINDS.index(kind), dim, n])
    m = 300 + n % 211
    db, qry = tie_case(kind, dim, n, m, rng)
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
