"""-m gpu: the fp16 candidate path's error bound, term by term, against the float64 reference (tests/fp16_keys_ref.py).

Bit-exact matching on the fp16 path rests on one inequality (DESIGN.md 2.1): for every candidate key,
|key value - real chunk-minimum distance| <= eps_pair + 2^(b-23) |key|.  Each case here checks its parts separately:
the operands bit for bit, the stats as upper bounds, the norm split of every row, the accumulation of every key against
the exact fp16 surrogate, and the statement the certification uses (every chunk outside keys 0..k-1 is no closer than
the lower bound of key k).  Then the certification's decisions end to end on near-ties built for each path."""
import numpy as np
import pytest

import fp16_keys_ref as ref
from regard3d_b200 import synth

pytestmark = pytest.mark.gpu


def _unit(g):
    return (g / np.maximum(np.linalg.norm(g, axis=1, keepdims=True), 1e-30)).astype(np.float32)


def _fp16_floor(x):
    """The largest fp16 value <= x (x > 0)."""
    h = np.float16(x)
    return h if np.float64(h) <= x else np.nextafter(h, np.float16(0))


def _rows(kind, n, dim, rng):
    if kind == "liop":                         # unit norm, all positive
        return _unit(np.abs(rng.standard_normal((n, dim))))
    if kind == "msurf":                        # unit norm, signed
        return _unit(rng.standard_normal((n, dim)))
    if kind == "sift":                         # float on a 0..255 scale, not integers
        return np.minimum(np.abs(rng.standard_normal((n, dim))) * 60.0, 255.0).astype(np.float32)
    if kind.startswith("dominant"):
        # a = (1, t, t, ...): the first product puts the running sum at about -2 (ulp 2^-22); every later product
        # -2 t^2 sits just under half an ulp (dominant_half) or just under one ulp (dominant_ulp) of it.  t is exact
        # in fp16, so the operands carry no quantisation error; half of the rows flip the signs of the small terms.
        f = 0.49 if kind == "dominant_half" else 0.99
        t = np.float64(_fp16_floor(np.sqrt(f * 2.0 ** -23)))
        a = np.full((n, dim), t)
        a[:, 0] = 1.0
        flip = rng.random((n, dim)) < 0.5
        flip[: n // 2] = False
        flip[:, 0] = False
        a[flip] = -t
        return a.astype(np.float32)
    if kind == "subnormal":                    # fp16 subnormals, and values below 2^-24 that fp16 flushes to zero
        a = rng.uniform(0, 2.0 ** -14, (n, dim)) * np.where(rng.random((n, dim)) < 0.5, -1, 1)
        tiny = rng.random((n, dim)) < 0.3
        a[tiny] = rng.uniform(0, 2.0 ** -25, tiny.sum())
        return a.astype(np.float32)
    if kind == "norm_under":                   # ||a||^2 just under the 2.6e8 cut (e0 = 15), one large component
        a = np.abs(rng.standard_normal((n, dim)))
        a[:, 0] = 40.0
        a = _unit(a).astype(np.float64) * np.sqrt(2.6e8 * rng.uniform(0.5, 0.9999, (n, 1)))
        a[0] *= np.sqrt(0.99985 / np.dot(a[0], a[0]) * 2.6e8)
        return a.astype(np.float32)
    if kind == "zero":                         # signed unit rows, every third one all zero
        a = _unit(rng.standard_normal((n, dim)))
        a[::3] = 0
        return a
    if kind == "u8":
        return rng.integers(0, 256, (n, dim)).astype(np.uint8)
    raise ValueError(kind)


def _pair_data(kind, dim, nI, nJ, seed):
    rng = np.random.default_rng(seed)
    if kind == "near_dup":                     # queries within 1e-4 of database rows: distance << norms
        db = _rows("liop", nI, dim, rng)
        q = db[rng.integers(0, nI, nJ)] + (1e-4 / np.sqrt(dim)) * rng.standard_normal((nJ, dim)).astype(np.float32)
        return db, q.astype(np.float32)
    if kind == "dup":                          # exact duplicates: zero distance, negative surrogate
        db = _rows("msurf", nI, dim, rng)
        return db, db[rng.integers(0, nI, nJ)].copy()
    db = _rows(kind, nI, dim, rng)
    q = _rows(kind, nJ, dim, rng)
    if kind == "zero":
        q[::4] = 0
    return db, q


def _xy(v, n):
    """Distinct keypoint positions of view v: the coordinate de-duplication keeps every distinct match."""
    return np.random.default_rng(1000 + v).uniform(0, 1000, (n, 2)).astype(np.float32)


def _upload(ctx, views):
    ctx.clear_regions()
    for v, d in enumerate(views):
        ctx.upload_regions(v, d, _xy(v, len(d)))


BOUND_CASES = [
    # (kind, D, nI, nJ); LIOP-144 at 2048 x 2048 is tests/test_gpu_match.py::test_candidate_error_bound_holds
    ("liop", 16, 255, 300), ("liop", 17, 256, 77), ("liop", 61, 257, 1000), ("liop", 64, 9, 130),
    ("liop", 129, 8, 2), ("liop", 224, 5000, 1001), ("liop", 240, 2, 333),
    ("msurf", 64, 5000, 2047), ("msurf", 240, 1000, 500), ("msurf", 17, 257, 129),
    ("sift", 128, 2048, 1000), ("sift", 224, 256, 300),
    ("near_dup", 144, 2048, 1500), ("near_dup", 240, 257, 300), ("near_dup", 16, 9, 50),
    ("dominant_half", 240, 256, 200), ("dominant_half", 64, 257, 100),
    ("dominant_ulp", 240, 256, 200), ("dominant_ulp", 144, 9, 100),
    ("subnormal", 144, 1000, 300), ("subnormal", 61, 255, 100),
    ("norm_under", 144, 1000, 500), ("norm_under", 240, 256, 100),
    ("dup", 144, 1000, 700), ("dup", 17, 8, 8),
    ("zero", 64, 1000, 300), ("zero", 240, 9, 20),
    ("u8", 72, 2048, 1000), ("u8", 200, 257, 500),
]


@pytest.mark.parametrize("kind,dim,nI,nJ", BOUND_CASES)
def test_candidate_error_bound_term_by_term(gpu_ctx, kind, dim, nI, nJ):
    db, q = _pair_data(kind, dim, nI, nJ, seed=dim * 7919 + nI)
    _upload(gpu_ctx, [db, q])
    out = ref.check_pair(gpu_ctx, 0, 1, db, q, "%s D=%d %dx%d" % (kind, dim, nI, nJ))
    if kind == "norm_under":
        assert gpu_ctx.debug_view_operands(0)["e0"] == 15
    if kind == "u8":
        assert out["quant"] != out["quant"] or out["quant"] == 0.0   # uint8 values are exact in fp16


def _small_exact_rows(rng, n, dim, radius):
    """Rows of norm about `radius` whose components are multiples of 2^-14 (exact in fp16)."""
    a = _unit(rng.standard_normal((n, dim))) * radius
    return (np.round(a * 2.0 ** 14) / 2.0 ** 14).astype(np.float32)


def _big_view(rng, n, dim):
    return _unit(np.abs(rng.standard_normal((n, dim)))) * np.float32(1.2e4)     # ||a||^2 ~ 1.44e8: e0 = 15


def _assert_matches_equal_oracle(ctx, oracle, descs, ratio, flags=0):
    """match_pairs over all pairs of the uploaded views equals the oracle's as ordered sequences; returns the count."""
    pairs = synth.exhaustive_pairs(len(descs))
    xys = [_xy(v, len(d)) for v, d in enumerate(descs)]
    ofs, m = oracle.match_pairs(descs, xys, pairs, ratio)
    got = ctx.match_pairs(pairs, ratio, flags).to_dict()
    for k, (I, J) in enumerate(pairs):
        e = m[int(ofs[k]):int(ofs[k + 1])]
        g = got.get((int(I), int(J)))
        g = np.zeros(0, e.dtype) if g is None else g
        assert np.array_equal(g["i"], e["i"]) and np.array_equal(g["j"], e["j"]), (I, J)
    return int(ofs[-1])


def _assert_neighbours_equal_oracle(ctx, oracle, I, J, db, q):
    idx, dist = ctx.search_neighbours(I, J, len(q))
    oi, od = oracle.search_neighbours(db, q)
    assert np.array_equal(idx, oi) and np.array_equal(dist.view(np.uint32), od.view(np.uint32))


def test_mixed_scales_share_one_exponent(gpu_ctx, oracle):
    """A view with norms near 1.2e4 sets e0 = 15 for the device; two views of norm 0.1 whose components are exact in
    fp16 are prepared under it: their p0 and p1 are fp16 subnormals, and the split error of such a row (up to
    2^(e0-36)) is several times the rest of their pair's bound."""
    rng = np.random.default_rng(31)
    big = _big_view(rng, 300, 144)
    db = _small_exact_rows(rng, 2048, 144, 0.1)
    q = (db[rng.integers(0, 2048, 1500)] + np.float32(2.0 ** -14) * rng.integers(-2, 3, (1500, 144))).astype(np.float32)
    _upload(gpu_ctx, [big, db, q])
    out = ref.check_pair(gpu_ctx, 1, 2, db, q, "mixed scales 0.1 beside 1.2e4")
    assert gpu_ctx.debug_view_operands(1)["e0"] == 15
    assert out["split_without_floor"] > 1.0       # the relative term alone does not cover these rows
    _assert_neighbours_equal_oracle(gpu_ctx, oracle, 1, 2, db, q)
    _assert_matches_equal_oracle(gpu_ctx, oracle, [big, db, q], 0.8)


def test_exponent_growth_reprepares_views_and_clear_resets_it(gpu_ctx, oracle):
    rng = np.random.default_rng(37)
    db = _small_exact_rows(rng, 1000, 64, 0.1)
    q = (db[rng.integers(0, 1000, 700)] + np.float32(2.0 ** -14) * rng.integers(-2, 3, (700, 64))).astype(np.float32)
    _upload(gpu_ctx, [db, q])
    _assert_matches_equal_oracle(gpu_ctx, oracle, [db, q], 0.8)
    e_small = gpu_ctx.debug_view_operands(0)["e0"]
    assert e_small == -3
    big = _big_view(rng, 300, 64)
    gpu_ctx.upload_regions(2, big, _xy(2, len(big)))
    o = gpu_ctx.debug_view_operands(0)                        # re-prepared under the grown exponent
    assert o["e0"] == 15
    rQ, rD = ref.prepare(db, 15)
    assert np.array_equal(o["opQ"].view(np.uint16), rQ.view(np.uint16)) and np.array_equal(o["opD"].view(np.uint16), rD.view(np.uint16))
    ref.check_pair(gpu_ctx, 0, 1, db, q, "after e0 growth -3 -> 15")
    _assert_matches_equal_oracle(gpu_ctx, oracle, [db, q, big], 0.8)
    _assert_neighbours_equal_oracle(gpu_ctx, oracle, 0, 1, db, q)
    _upload(gpu_ctx, [db, q])                                 # clear_regions: the exponent starts over
    assert gpu_ctx.debug_view_operands(0)["e0"] == e_small
    ref.check_pair(gpu_ctx, 0, 1, db, q, "after clear_regions")


@pytest.mark.parametrize("case", ["norm_over_cut", "components_32000"])
def test_views_beyond_the_fp16_operands_take_the_exact_scan(gpu_ctx, oracle, case):
    rng = np.random.default_rng(41)
    n, dim = 600, 144
    if case == "norm_over_cut":                # ||a||^2 just over 2.6e8
        a = _unit(np.abs(rng.standard_normal((n, dim)))).astype(np.float64) * np.sqrt(2.61e8)
    else:                                      # one component at +-32000 per row (the operand range's edge)
        a = np.abs(rng.standard_normal((n, dim))) * 50.0
        a[:, 0] = 32000.0 * np.where(rng.random(n) < 0.5, -1, 1)
    descs = [a.astype(np.float32)]
    descs.append((descs[0][rng.permutation(n)] + rng.standard_normal((n, dim)).astype(np.float32) * 20).astype(np.float32))
    _upload(gpu_ctx, descs)
    assert gpu_ctx.debug_view_operands(0)["opD"] is None
    assert _assert_matches_equal_oracle(gpu_ctx, oracle, descs, 0.8) > 100
    _assert_neighbours_equal_oracle(gpu_ctx, oracle, 0, 1, descs[0], descs[1])


@pytest.mark.parametrize("dim", [50, 61, 130])
def test_u8_rows_not_a_multiple_of_four_bytes(gpu_ctx, oracle, dim):
    """uint8 views with D % 4 != 0 use neither the integer path (D % 16 != 0) nor the binned re-rank, which reads rows
    in 4-byte words: they are matched by the exact scan."""
    rng = np.random.default_rng(dim)
    n = 900
    db = rng.integers(0, 256, (n, dim)).astype(np.uint8)
    q = np.clip(db[rng.permutation(n)].astype(int) + rng.integers(-6, 7, (n, dim)), 0, 255).astype(np.uint8)
    q[::3] = rng.integers(0, 256, (len(q[::3]), dim))
    a, b = db.astype(np.float64), q.astype(np.float64)          # exact integer distances
    d3 = np.sort((b * b).sum(1)[:, None] + (a * a).sum(1)[None, :] - 2.0 * b @ a.T, 1)[:, :3]
    q = q[(d3[:, 0] < d3[:, 1]) & (d3[:, 1] < d3[:, 2])]         # no exact ties (their order is std::partial_sort's)
    _upload(gpu_ctx, [db, q])
    assert _assert_matches_equal_oracle(gpu_ctx, oracle, [db, q], 0.8) > 100
    _assert_neighbours_equal_oracle(gpu_ctx, oracle, 0, 1, db, q)


# ---- certification decisions end to end --------------------------------------------------------------------------

def _two_squares(limit):
    t = {}
    for x in range(limit + 1):
        for y in range(x + 1):
            t.setdefault(x * x + y * y, (x, y))
    return t


def _offset_with_norm2(target, dim, rng, cap, two_sq):
    """An integer vector e (|e_k| <= cap) with sum e_k^2 == target exactly."""
    while True:
        e = np.zeros(dim, np.int64)
        per = target / (dim - 4)
        c = max(1, min(cap, int(np.sqrt(3 * per))))
        e[:dim - 4] = rng.integers(-c, c + 1, dim - 4)
        rest = target - int((e * e).sum())
        if rest < 0:
            continue
        for x in range(min(cap, int(np.sqrt(rest))), -1, -1):
            r2 = rest - x * x
            for y in range(min(x, int(np.sqrt(r2))), -1, -1):
                hit = two_sq.get(r2 - y * y)
                if hit and max(hit) <= cap:
                    e[dim - 4:] = [x, y, hit[0], hit[1]]
                    return e * np.where(rng.random(dim) < 0.5, -1, 1)


def test_ratio_boundary_and_early_rejection_on_exact_keys(gpu_ctx, oracle):
    """uint8 D = 128 (integer path: eps_pair = 0, the key error is the chunk-id packing alone).  Per planted query,
    d2 = 16 m and d1 = 9 m - 1, 9 m or 9 m + 1 around fl(0.75^2 d2) = 9 m exactly: the strict ratio test passes only
    for the first.  With 10 chunk bits the packing moves a key by up to 2^-13 of its value, far more than the gap:
    early rejection must keep its margin for it.  Unplanted queries (d1 ~ d2) are rejected early."""
    rng = np.random.default_rng(43)
    dim, nI, n_plant = 128, 5000, 600
    two_sq = _two_squares(63)
    db = rng.integers(0, 256, (nI, dim)).astype(np.int64)
    q = rng.integers(64, 192, (n_plant + 200, dim)).astype(np.int64)
    rows = rng.permutation(nI)[:2 * n_plant].reshape(n_plant, 2)
    want = []
    for j in range(n_plant):
        m = int(rng.integers(9000, 11000))
        s = (j % 3) - 1
        for row, target in ((rows[j, 0], 9 * m + s), (rows[j, 1], 16 * m)):
            db[row] = q[j] + _offset_with_norm2(target, dim, rng, 63, two_sq)
        want.append(s < 0)
    db, q = db.astype(np.uint8), q.astype(np.uint8)
    _upload(gpu_ctx, [db, q])
    n = _assert_matches_equal_oracle(gpu_ctx, oracle, [db, q], 0.75)
    t = gpu_ctx.match_timing()
    assert n >= sum(want) and t["rejected_queries"] > 0, (n, t)


def _l2_f32(q, db):
    """Squared L2 in float32 in the oracle's order (4-way unrolled, openMVG::matching::L2; dim % 4 == 0), nq x n."""
    acc = np.zeros((len(q), len(db)), np.float32)
    for k in range(0, q.shape[1], 4):
        d = q[:, None, k:k + 4] - db[None, :, k:k + 4]
        acc = acc + (((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]) + d[..., 3] * d[..., 3])
    return acc


@pytest.mark.parametrize("nI,nJ", [(2048, 1500), (2048, 3000), (20, 500)])
def test_near_equidistant_rows_reach_stage_b_and_the_exact_scan(gpu_ctx, oracle, nI, nJ):
    """Database rows on the unit sphere, queries within 1e-5 of its centre: every row is at distance 1 +- a few eps_pair,
    so third and sixth keys fall within eps of E2 (stage B, then the exact scan).  3000 queries send more than 2048 items
    to the exact scan (one block per item).  20 database rows are three real chunks: stage B bounds them with a padding
    key and certifies, and the exact scan of every query (R3D_MATCH_EXACT_SCAN) leaves most of its 32 row slices empty."""
    rng = np.random.default_rng(nI + nJ)
    dim = 64
    db = _unit(rng.standard_normal((nI, dim)))
    q = (1e-5 * _unit(rng.standard_normal((nJ + nJ // 4, dim)))).astype(np.float32)
    # Upstream orders equal float distances as std::partial_sort leaves them, not by index: keep the near-ties, drop
    # the queries whose three smallest float distances are not distinct
    d3 = np.sort(_l2_f32(q, db), 1)[:, :3]
    assert _l2_f32(q[:1], db[:1])[0, 0] == np.float32(oracle.l2(q[0], db[0]))
    q = q[(d3[:, 0] < d3[:, 1]) & (d3[:, 1] < d3[:, 2])][:nJ]
    assert len(q) == nJ
    _upload(gpu_ctx, [db, q])
    _assert_neighbours_equal_oracle(gpu_ctx, oracle, 0, 1, db, q)
    fb = gpu_ctx.match_timing()["fallback_queries"]
    assert _assert_matches_equal_oracle(gpu_ctx, oracle, [db, q], 1.0) > 0
    t = gpu_ctx.match_timing()
    assert t["third_chunk_queries"] > 0, t
    if nI > 32:
        assert fb > (2048 if nJ > 2048 else 0) and t["fallback_queries"] > 0, (fb, t)
    else:
        _assert_matches_equal_oracle(gpu_ctx, oracle, [db, q], 1.0, flags=1)   # R3D_MATCH_EXACT_SCAN
        assert gpu_ctx.match_timing()["fallback_queries"] == nJ
