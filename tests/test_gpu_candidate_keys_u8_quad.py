"""-m gpu: integer candidate keys where the quad bound decides.  Lane q of a quad tests the chunks c = q (mod 4) of each
row and rejects chunks against a bound taken from all four lanes' key sets, so rows whose nearest chunks all sit in one
lane's quarter (or split 5/1, 3/3) make the other lanes reject almost everything.  numpy predicts the whole key array
bit for bit (test_gpu_candidate_keys_u8.expected_keys)."""
import numpy as np
import pytest

from test_gpu_candidate_keys_u8 import CHUNK, NUM_KEYS, expected_keys

pytestmark = pytest.mark.gpu

# lanes of the NUM_KEYS nearest chunks of a row, as offsets from a per-row lane a: all in a, 5 in a and 1 in a + 1, ...
PATTERNS = {"one_lane": [0] * 6, "five_one": [0] * 5 + [1], "three_three": [0] * 3 + [2] * 3}


def planted_case(pattern, dim, n, m, rng):
    """Random database and queries; each query row gets NUM_KEYS near database rows in distinct chunks of the pattern's
    lanes and three runner-up rows in the other lanes, each planted row used by one query only."""
    db = rng.integers(0, 256, (n, dim)).astype(np.uint8)
    qry = rng.integers(0, 256, (m, dim)).astype(np.uint8)
    nchunks = (n + CHUNK - 1) // CHUNK
    free = [list(range(CHUNK * c, min(CHUNK * c + CHUNK, n))) for c in range(nchunks)]

    def plant(row, lane, ncols, lo, hi, used):
        cands = [c for c in range(lane, nchunks, 4) if free[c] and c not in used]
        c = int(rng.choice(cands))
        used.add(c)
        r = free[c].pop(int(rng.integers(len(free[c]))))
        a = qry[row].astype(np.int64)
        cols = rng.choice(dim, ncols, replace=False)
        a[cols] += np.where(a[cols] < 128, 1, -1) * rng.integers(lo, hi + 1, ncols)   # no clipping
        db[r] = a

    for row in range(m):
        a = row % 4
        used = set()
        lanes = [(a + d) % 4 for d in PATTERNS[pattern]]
        for lane in lanes:               # squared distance 1 .. 2700
            plant(row, lane, int(rng.integers(1, 4)), 1, 30, used)
        others = [x for x in range(4) if x not in lanes]
        for k in range(3):               # 4800 .. 10800
            plant(row, others[k % len(others)], 3, 40, 60, used)
    return db, qry


@pytest.mark.parametrize("pattern", sorted(PATTERNS))
@pytest.mark.parametrize("dim,n", [(64, 3001), (128, 5000), (256, 2600)])
def test_integer_candidate_keys_quad_bound_bit_exact(gpu_ctx, pattern, dim, n):
    rng = np.random.default_rng([sorted(PATTERNS).index(pattern), dim, n])
    m = 97 + n % 61
    db, qry = planted_case(pattern, dim, n, m, rng)
    gpu_ctx.clear_regions()
    gpu_ctx.upload_regions(0, db, rng.uniform(0, 500, (n, 2)).astype(np.float32))
    gpu_ctx.upload_regions(1, qry, rng.uniform(0, 500, (m, 2)).astype(np.float32))
    keys, eps = gpu_ctx.debug_candidate_keys(0, 1, m)
    assert eps == 0.0
    exp = expected_keys(db, qry)
    bits = max(4, int(np.ceil(np.log2((n + 255) // 256 * 256 // CHUNK))))
    lanes = np.sort((exp[:, :NUM_KEYS] & np.uint32((1 << bits) - 1)) % 4, 1)
    want = np.sort((np.arange(m)[:, None] + np.array(PATTERNS[pattern])[None, :]) % 4, 1)
    assert np.array_equal(lanes, want), "the planted chunks are not the nearest"
    got = keys[:m]
    bad = np.nonzero((got != exp).any(1))[0]
    assert np.array_equal(got, exp), "%d of %d query rows differ, first row %d: got %s expected %s" % (
        bad.size, m, bad[0], got[bad[0]].tolist(), exp[bad[0]].tolist())
