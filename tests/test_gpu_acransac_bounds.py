"""-m gpu: the AC-RANSAC kernel's tier-1 bounds and tier-2 NFA scan (k_acransac_fused, through the same device code in
r3d_debug_acransac_score) against exact rational residuals and a float64 NFA with exact log10 binomials
(tests/acransac_ref.py), on all four models.

Tier 1 may only skip a model whose best NFA cannot beat the best so far.  That holds when, for every model:
  1. lo <= e <= hi for the tier-2 residual e and for the exact one;
  2. cnt_lo <= #{e <= max_thr} <= cnt_hi;
  3. lb <= the tier-2 NFA (+inf when cnt_hi <= the minimal sample);
and the tier-2 scan itself is right when
  4. err is the k-th smallest tier-2 residual;
  5. nfa / k are the reference minimum / argmin (up to the float tables' error and a few ulp per term);
  6. the float log-combination tables stay within the error bound the kernel subtracts.
1-4 are exact assertions.  The inputs are the ones where kernels go wrong: RANSAC models from inlier and outlier
samples, cancellation (exact fits, epipoles, the line at infinity, entries over 16 decades, NaN / inf), extreme scales,
residuals on bin edges and ties, and every size class boundary."""
import math
from fractions import Fraction

import numpy as np
import pytest

import acransac_ref as ref
from oracle import pyoracle as po
from oracle import pyoracle_resection as pro
from relpose_scenes import two_view
from resection_scenes import make_view, rodrigues

pytestmark = pytest.mark.gpu

W, H = 1920, 1080
EXACT_BUDGET = 1500  # exact rational residuals per case (a sample of the (model, point) grid above that)


# ---- the filters' adaptors: coordinates, squared precision bound and logalpha0 of each model -------------------------
def _norm(x, w, h):
    s = 1.0 / math.sqrt(w * h)
    return np.c_[s * x[:, 0] + (-0.5 * w) * s, s * x[:, 1] + (-0.5 * h) * s], s


def _logalpha0(model, w, h, s=1.0):
    D, A = math.hypot(w, h), float(w) * h
    return {0: math.log10(2 * D / A / s), 1: math.log10(math.pi / A / (s * s)), 2: math.log10(2 * D / A * 0.5),
            3: math.log10(math.pi / A)}[model]


def _F_from_E(E, K1, K2):
    def kinv(K):
        f, px, py = K[:3]
        return np.array([[1 / f, 0, -px / f], [0, 1 / f, -py / f], [0, 0, 1.0]])
    return kinv(K2).T @ E @ kinv(K1)


def _skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]], float)


def _bearing(K, x):
    b = np.c_[(x[:, 0] - K[1]) / K[0], (x[:, 1] - K[2]) / K[0], np.ones(len(x))]
    return b / np.linalg.norm(b, axis=1)[:, None]


# ---- the checks ---------------------------------------------------------------------------------------------------
def _check(ctx, model, x1, x2, models, max_thr, logalpha0, K=(0,) * 6, x3=None, nfa_ref=True, seed=0):
    ns = ref.MIN_SAMPLES[model]
    x1 = np.ascontiguousarray(x1, np.float64)
    x2 = np.ascontiguousarray(x2, np.float64)
    models = np.ascontiguousarray(models, np.float64).reshape(-1, ref.MODEL_SIZE[model])
    M, n = len(x1), len(models)
    r = ctx.debug_acransac_score(model, x1, x2, models, max_thr, logalpha0, K, x3=x3, per_point=True)
    sc, lo, hi, e = r["score"], r["lo"], r["hi"], r["e"]
    # 1. the tier-1 interval holds the tier-2 residual ...
    fin = np.isfinite(e)
    bad = fin & ~((lo <= e) & (e <= hi))
    assert not bad.any(), "tier-1 interval misses the tier-2 residual at (model, point) %s: lo %r e %r hi %r" % (
        np.argwhere(bad)[0], lo[bad][0], e[bad][0], hi[bad][0])
    # ... and the exact one
    rng = np.random.default_rng(seed)
    cells = [(m, i) for m in range(n) for i in range(M)]
    if len(cells) > EXACT_BUDGET:
        cells = [cells[j] for j in rng.choice(len(cells), EXACT_BUDGET, replace=False)]
    for m, i in cells:
        ex = ref.exact_residual(model, models[m], x1[i], x2[i], 0.0 if x3 is None else x3[i])
        if ex is None:
            continue
        assert Fraction(lo[m, i]) <= ex and (hi[m, i] == np.inf or ex <= Fraction(hi[m, i])), \
            "tier-1 interval misses the exact residual at (%d, %d): lo %r exact %r hi %r" % (m, i, lo[m, i], float(ex), hi[m, i])
    for m in range(n):
        s = sc[m]
        inl = e[m][e[m] <= max_thr]
        # 2. counts
        assert s["count"] == len(inl)
        assert s["cnt_lo"] <= s["count"] <= s["cnt_hi"], (m, s)
        # 3. the lower bound
        assert s["lb"] <= s["nfa"], (m, s)
        if s["cnt_hi"] <= ns:
            assert s["nfa"] == np.inf, (m, s)
        # 4. errorMax
        if s["k"] > ns:
            assert s["err"] == np.sort(inl)[s["k"] - 1], (m, s)
        else:
            assert s["nfa"] == np.inf and s["err"] == 0.0, (m, s)
    _check_tables(r, model, M)
    if nfa_ref:
        _check_nfa(r, model, x1, x2, x3, models, max_thr, logalpha0)
    return r


def _check_tables(r, model, M):
    ns = ref.MIN_SAMPLES[model]
    lcn, lck = r["logc_n"].astype(np.float64), r["logc_k"].astype(np.float64)
    bound = lcn[M + 1]
    exact = np.array([ref.log10_binom(M, k) for k in range(M + 1)])
    err = np.abs(lcn[:M + 1] - exact)
    assert (err <= bound).all(), "logc_n[%d] off by %r > its bound %r" % (int(err.argmax()), err.max(), bound)
    if M > ns:
        kk = np.arange(ns + 1, M + 1)
        ek = np.abs(lck[kk] - np.array([ref.log10_binom(int(k), ns) for k in kk]))
        assert 2 * ek.max() <= 1e-4, "logc_k error %r: twice it exceeds the fixed slack of the lower bound" % ek.max()
    return bound


def _check_nfa(r, model, x1, x2, x3, models, max_thr, logalpha0):
    ns = ref.MIN_SAMPLES[model]
    M = len(x1)
    lcn, lck = r["logc_n"].astype(np.float64), r["logc_k"].astype(np.float64)
    # the float tables' measured error at every k the scan can use (not the stored bound, which is far looser)
    tbl_err = np.zeros(M + 1)
    if M > ns:
        kk = np.arange(ns + 1, M + 1)
        tbl_err[kk] = (np.abs(lcn[kk] - np.array([ref.log10_binom(M, int(k)) for k in kk]))
                       + np.abs(lck[kk] - np.array([ref.log10_binom(int(k), ns) for k in kk])))
    for m, s in enumerate(r["score"]):
        res = ref.float_residuals(model, models[m], x1, x2, x3)
        curve = ref.nfa_curve(model, res, M, max_thr, logalpha0)
        best, kbest = ref.best_nfa(curve)
        if kbest is None:
            assert s["nfa"] == np.inf, (m, s)
            continue
        # a few ulp per term of every NFA(k), plus the tables' error where the two minima are taken
        tol = tbl_err[ns + 1:max(curve) + 1].max() + 1e-13 * ref.nfa_term_scale(model, res, M, max_thr, logalpha0)
        assert abs(s["nfa"] - best) <= tol, (m, s["nfa"], best, tol)
        assert s["k"] == kbest or (int(s["k"]) in curve and curve[int(s["k"])] <= best + 2 * tol), (m, s["k"], kbest)


# ---- inputs -------------------------------------------------------------------------------------------------------
def _scene(M, seed, outlier_frac=0.4, f=None, w=W, h=H, baseline=(1.0, 0.1, 0.05)):
    xI, xJ, R, t, K = two_view(M, seed, outlier_frac=outlier_frac, f=f, w=w, h=h, baseline=baseline)
    xI, xJ = xI.astype(np.float64), xJ.astype(np.float64)
    Ft = _F_from_E(_skew(t) @ R, K, K)
    inl = ref.float_residuals(2, Ft.ravel(), xI, xJ) < 4.0
    return xI, xJ, K, inl


def _ransac_models(model, n_models, xI, xJ, K, inl, seed, x3=None):
    """n_models models of the given kind from minimal samples, alternately drawn among the inliers and the outliers."""
    rng = np.random.default_rng(seed)
    ns = ref.MIN_SAMPLES[model]
    pools = [np.nonzero(inl)[0], np.nonzero(~inl)[0]]
    pools = [p for p in pools if len(p) >= ns] or [np.arange(len(xI))]
    out, tries = [], 0
    while len(out) < n_models and tries < 50 * n_models:
        pool = pools[tries % len(pools)]
        tries += 1
        idx = rng.choice(pool, ns, replace=False)
        if model == 0:
            got = [F.ravel() for F in po.seven_point(xI[idx], xJ[idx])]
        elif model == 1:
            Hm = po.four_point(xI[idx], xJ[idx])
            got = [] if Hm is None else [Hm.ravel()]
        elif model == 2:
            got = [_F_from_E(E, K, K).ravel() for E in po.five_point(_bearing(K, xI[idx]), _bearing(K, xJ[idx]))]
        else:
            X = np.c_[xI[idx], x3[idx]]
            got = [P.ravel() for P in pro.p3p(K[:3], X, xJ[idx])]
        out.extend(got)
    assert len(out) >= n_models
    return np.array(out[:n_models])


def _case_pair(model, M, n_models, seed, outlier_frac=0.4, precision=4.0):
    """A two-view pair (models 0-2) or a view with known structure (model 3) and RANSAC models on it."""
    if model == 3:
        v = make_view(seed, M, model=1, outliers=outlier_frac)
        K = np.array([v["focal"], v["ppx"], v["ppy"], float(v["width"]) ** 2 + float(v["height"]) ** 2, 0.0, 0.0])
        P = K[:3]
        Kt = np.array([[P[0], 0, P[1]], [0, P[0], P[2]], [0, 0, 1.0]]) @ np.c_[v["R"], v["t"]]
        inl = ref.float_residuals(3, Kt.ravel(), v["X"][:, :2], v["x"], v["X"][:, 2]) < 4.0
        models = _ransac_models(3, n_models, v["X"][:, :2], v["x"], K, inl, seed, x3=v["X"][:, 2])
        return dict(model=3, x1=v["X"][:, :2], x2=v["x"], x3=v["X"][:, 2], models=models, max_thr=precision ** 2,
                    logalpha0=_logalpha0(3, v["width"], v["height"]), K=K)
    xI, xJ, K, inl = _scene(M, seed, outlier_frac)
    if model == 2:
        models = _ransac_models(2, n_models, xI, xJ, K, inl, seed)
        return dict(model=2, x1=xI, x2=xJ, models=models, max_thr=precision ** 2, logalpha0=_logalpha0(2, W, H),
                    K=np.r_[K, K])
    a, s = _norm(xI, W, H)
    b, _ = _norm(xJ, W, H)
    models = _ransac_models(model, n_models, a, b, K, inl, seed)
    return dict(model=model, x1=a, x2=b, models=models, max_thr=precision ** 2 * s * s, logalpha0=_logalpha0(model, W, H, s))


def _run(ctx, c, **kw):
    return _check(ctx, c["model"], c["x1"], c["x2"], c["models"], c["max_thr"], c["logalpha0"], c.get("K", (0,) * 6),
                  x3=c.get("x3"), **kw)


# ---- RANSAC models, sizes and group occupancy ---------------------------------------------------------------------
@pytest.mark.parametrize("model", [0, 1, 2, 3])
@pytest.mark.parametrize("n_models", [1, 7, 8, 23])
def test_ransac_models(gpu_ctx, model, n_models):
    # groups of 7 models (one per consumer warp): full, partial, and spread over several iterations of MAX_MODELS
    _run(gpu_ctx, _case_pair(model, 400, n_models, seed=10 * model + n_models), seed=n_models)


@pytest.mark.parametrize("model", [0, 1, 2, 3])
def test_sizes(gpu_ctx, model):
    ns = ref.MIN_SAMPLES[model]
    for M in (ns, ns + 1, 31, 32, 33, 224, 225, 256, 257, 1024, 1025):
        c = _case_pair(model, max(M, 40), 8, seed=M, outlier_frac=0.3)
        for k in ("x1", "x2", "x3"):
            if k in c:
                c[k] = c[k][:M]
        _run(gpu_ctx, c, seed=M)


@pytest.mark.parametrize("model", [0, 1, 2, 3])
def test_huge_boundary(gpu_ctx, model):
    # 16384: the largest shared-memory sort; 16385: the global-scratch (HUGE) instantiation
    for M in (16384, 16385):
        _run(gpu_ctx, _case_pair(model, M, 7, seed=M + model, outlier_frac=0.5), seed=M)


@pytest.mark.parametrize("model", [0, 1, 2, 3])
def test_table_bounds_large(gpu_ctx, model):
    # logc_n within its stored bound, and twice the logc_k error inside the fixed 1e-4 slack, at M = 40 000
    c = _case_pair(model, 40000, 1, seed=40000 + model, outlier_frac=0.5)
    r = gpu_ctx.debug_acransac_score(c["model"], c["x1"], c["x2"], c["models"], c["max_thr"], c["logalpha0"],
                                     c.get("K", (0,) * 6), x3=c.get("x3"))
    assert r["score"]["lb"][0] <= r["score"]["nfa"][0]
    _check_tables(r, model, 40000)


# ---- cancellation -------------------------------------------------------------------------------------------------
def _epipolar_points(e, rng, n, scale=1.0):
    """Integer points x1 and x2 = e + lam (x1 - e), lam dyadic: x2^T [e]x x1 = 0 exactly in double."""
    x1 = rng.integers(-40, 40, (n, 2)).astype(float) * scale
    lam = rng.integers(-8, 9, n) / 4.0
    x2 = e[:2] + lam[:, None] * (x1 - e[:2])
    return x1, x2


def _spread_models(rng, n, size):
    return rng.choice([-1.0, 1.0], (n, size)) * 10.0 ** rng.uniform(-8, 8, (n, size))


def _ulp_walk(p, rng, n):
    """n points at p, a few ulp from it in each coordinate, and at relative distances 2^-50 .. 2^-10 from it."""
    j = rng.integers(-16, 17, (n, 2))
    k = rng.integers(10, 51, (n, 1))
    out = p + j * np.spacing(np.abs(p))
    far = rng.random(n) < 0.5
    out[far] = p * (1 + rng.choice([-1.0, 1.0], (far.sum(), 2)) * 2.0 ** -k[far].astype(float))
    out[:4] = p
    return out


@pytest.mark.parametrize("model", [0, 2])
def test_epipolar_cancellation(gpu_ctx, model):
    rng = np.random.default_rng(5 + model)
    # an integer epipole under an integer skew F: x2^T F x1 = 0 exactly in double at dyadic points of the epipolar lines
    e = np.array([3.0, 5.0, 1.0])
    F = _skew(e)
    x1, x2 = _epipolar_points(e, rng, 300)
    x2[100:150] += 2.0 ** -30                                   # next to an exact fit
    x2[150:200, 1] += rng.uniform(-1, 1, 50)                    # ordinary residuals
    x1[200:210], x2[210:220] = e[:2], e[:2]                     # on the epipoles (A or B = 0 exactly)
    models = [F, F * 2.0 ** -20, F * 2.0 ** 20, F + np.diag([2.0 ** -40, 0, 0])]
    models = np.r_[np.array(models).reshape(-1, 9), _spread_models(rng, 3, 9)]
    _check(gpu_ctx, model, x1, x2, models, 1.0, -2.0, K=(1000.0, 0, 0, 1000.0, 0, 0), nfa_ref=False)
    # a generic rank-2 F = [e2]x Mx (non-dyadic entries): at and next to its epipoles e1 = Mx^-1 e2 and e2, F x1 and
    # F^T x2 vanish only up to rounding, so A and B reach 0 through cancellation
    e2 = np.array([123.456789, -45.6789012, 1.0])
    Mx = np.eye(3) + 0.1 * rng.standard_normal((3, 3))
    G = _skew(e2) @ Mx
    e1 = np.linalg.solve(Mx, e2)
    e1 = e1[:2] / e1[2]
    n = 600
    x1 = np.r_[_ulp_walk(e1, rng, n // 2), e1 + rng.uniform(-200, 200, (n // 2, 2))]
    x2 = np.r_[e2[:2] + rng.uniform(-200, 200, (n // 4, 2)), _ulp_walk(e2[:2], rng, n // 2),
               e2[:2] + rng.uniform(-200, 200, (n // 4, 2))]
    models = np.r_[G.ravel()[None], (G * 1e-7).ravel()[None], (G * 3e5).ravel()[None]]
    _check(gpu_ctx, model, x1, x2, models, 1.0, -2.0, K=(1000.0, 0, 0, 1000.0, 0, 0), nfa_ref=False)


@pytest.mark.parametrize("model", [0, 2])
def test_epipolar_rounding_extremes(gpu_ctx, model):
    """Points on the epipolar lines of a model whose entries all sit just below +-2, near the corners of the coordinate
    box: the terms of x2^T F x1 are as large as eta assumes, and the 256 points kept are those where the tier-2
    evaluation of it strays furthest from its exact value (found against long double)."""
    rng = np.random.default_rng(17 + model)
    F = rng.choice([-1.0, 1.0], (3, 3)) * (2 - rng.uniform(0, 1e-3, (3, 3)))
    R, n = 1024.0 - 2.0 ** -40, 400000
    a = rng.choice([-1, 1], (n, 2)) * rng.uniform(0.97 * R, R, (n, 2))
    l = np.c_[a, np.ones(n)] @ F.T
    x = rng.choice([-1, 1], n) * rng.uniform(0.97 * R, R, n)
    y = -(l[:, 0] * x + l[:, 2]) / l[:, 1]
    ok = np.abs(y) <= R
    a, b = a[ok], np.c_[x[ok], y[ok]]
    fx = [F[r, 0] * a[:, 0] + F[r, 1] * a[:, 1] + F[r, 2] for r in range(3)]
    y2 = b[:, 0] * fx[0] + b[:, 1] * fx[1] + fx[2]
    L = np.longdouble
    fl = [L(F[r, 0]) * a[:, 0].astype(L) + L(F[r, 1]) * a[:, 1].astype(L) + L(F[r, 2]) for r in range(3)]
    yl = b[:, 0].astype(L) * fl[0] + b[:, 1].astype(L) * fl[1] + fl[2]
    keep = np.argsort(-np.abs(y2.astype(L) - yl))[:256]
    _check(gpu_ctx, model, a[keep], b[keep], F.ravel()[None], 1e-6, -3.0, nfa_ref=False)


def test_line_at_infinity(gpu_ctx):
    rng = np.random.default_rng(7)
    # a projective row with non-dyadic entries: on y0 = -(a x + c) / b, hw = a x + b y0 + c is rounding noise of either
    # sign; a few ulp of y0 away it is tiny and signed, and relative offsets 2^-46 .. 2^-4 walk it across q < 1e-3
    a, b, c = 0.123456789, 0.0987654321, 1.0
    Hm = np.array([[1.0, 0, 0], [0, 1.0, 0], [a, b, c]])
    M = 500
    x1 = rng.uniform(-60, 60, (M, 2))
    y0 = -(a * x1[:, 0] + c) / b
    j = rng.integers(-8, 9, M)
    k = rng.integers(4, 47, M).astype(float)
    y = np.where(rng.random(M) < 0.5, y0 + j * np.spacing(np.abs(y0)), y0 * (1 + rng.choice([-1.0, 1.0], M) * 2.0 ** -k))
    y[:40] = y0[:40]
    x1[:400, 1] = y[:400]                                       # the last 100 points: ordinary ones
    x2 = x1 + rng.uniform(-2, 2, (M, 2))
    models = np.r_[Hm.ravel()[None], (Hm * 2.0 ** 30).ravel()[None], (Hm * 3e-5).ravel()[None], _spread_models(rng, 5, 9)]
    _check(gpu_ctx, 1, x1, x2, models, 4.0, -3.0, nfa_ref=False)


@pytest.mark.parametrize("model", [0, 1, 2, 3])
def test_degenerate_models(gpu_ctx, model):
    """NaN and +-inf entries, an all-zero model, entries spread over 1e-8 .. 1e8: any interval must still hold."""
    c = _case_pair(model, 300, 4, seed=77 + model)
    ms = ref.MODEL_SIZE[model]
    rng = np.random.default_rng(model)
    odd = [np.zeros(ms)]
    for v in (np.nan, np.inf, -np.inf):
        m = c["models"][0].copy()
        m[rng.integers(ms)] = v
        odd.append(m)
    c["models"] = np.r_[c["models"], np.array(odd), _spread_models(rng, 8, ms)]
    sc = _run(gpu_ctx, c, nfa_ref=False)["score"]
    assert sc["count"][4] == 0 and sc["nfa"][4] == np.inf  # the all-zero model: every residual is 0 / 0


# ---- scale --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f", [1e2, 1e3, 1e4, 1e5])
def test_essential_scale(gpu_ctx, f):
    # a 10 000 x 10 000 pixel pair: points back-projected from view I at depths 5 .. 15, seen from a moved view J
    w = h = 10000
    rng = np.random.default_rng(int(f))
    K = np.array([f, w / 2.0, h / 2.0])
    n = 500
    u, v, z = rng.uniform(0, w, n), rng.uniform(0, h, n), rng.uniform(5, 15, n)
    X = np.c_[(u - K[1]) / f * z, (v - K[2]) / f * z, z]
    R, t = rodrigues(np.array([0.01, -0.02, 0.005])), np.array([0.3, 0.05, 0.02])
    Xj = X @ R.T + t
    xI = np.c_[u, v]
    xJ = f * Xj[:, :2] / Xj[:, 2:3] + K[1:] + rng.normal(size=(n, 2)) * 0.5
    bad = rng.random(n) < 0.4
    xJ[bad] = rng.uniform(0, w, (bad.sum(), 2))
    models = _ransac_models(2, 8, xI, xJ, K, ~bad, int(f))
    _check(gpu_ctx, 2, xI, xJ, models, 4.0, _logalpha0(2, w, h), K=np.r_[K, K], seed=int(f))


@pytest.mark.parametrize("scale", [1e-3, 1.0, 1e3, 1e6])
@pytest.mark.parametrize("precision", [0.5, np.inf])
def test_resection_scale(gpu_ctx, scale, precision):
    v = make_view(int(scale * 10) % 997, 400, model=1, outliers=0.3)
    X = v["X"] * scale
    X[:20] = 2 * (v["C"] * scale) - X[:20]                      # behind the camera
    K = np.array([v["focal"], v["ppx"], v["ppy"], 1.0 if precision == np.inf else 4e6, 0.0, 0.0])
    Kt = np.array([[K[0], 0, K[1]], [0, K[0], K[2]], [0, 0, 1.0]])
    Pt = Kt @ np.c_[v["R"], v["t"] * scale]
    inl = ref.float_residuals(3, Pt.ravel(), X[:, :2], v["x"], X[:, 2]) < 4.0
    models = np.r_[Pt.ravel()[None], _ransac_models(3, 11, X[:, :2], v["x"], K, inl, 3, x3=X[:, 2])]
    # an infinite bound with a tiny top-bin start (K[3] = 1): almost every residual is clamped into the top bin
    _check(gpu_ctx, 3, X[:, :2], v["x"], models, precision ** 2, _logalpha0(3, v["width"], v["height"]), K=K, x3=X[:, 2])


# ---- bins and ties: identity homographies and integer offsets, scaled by powers of two ----------------------------
def _offsets_case(rng, d, p, n_models=8):
    """x2 = x1 + d 2^-p: residuals (dx^2 + dy^2) 2^-2p exactly; models shift by dyadic translations."""
    M = len(d)
    x1 = rng.integers(-64, 64, (M, 2)).astype(float)
    x2 = x1 + d * 2.0 ** -p
    models = []
    for j in range(n_models):
        T = np.eye(3)
        T[:2, 2] = np.array([j % 3 - 1, j // 3 - 1]) * 2.0 ** -p
        models.append((T * 2.0 ** (j % 4)).ravel())              # a power-of-two multiple: the same residuals
    return x1, x2, np.array(models)


@pytest.mark.parametrize("p", [0, 10, 30])
def test_bin_edges_and_threshold(gpu_ctx, p):
    rng = np.random.default_rng(p)
    # dx^2 + dy^2 in {1, 2, 4, ..., 32, 34, 36, 40, 41, 45, 50}: lower edges of bins (5 mantissa bits); 50 = the bound
    edges = np.array([(1, 0), (1, 1), (2, 0), (2, 2), (4, 0), (4, 4), (5, 3), (6, 0), (6, 2), (5, 4), (6, 3), (5, 5)])
    d = edges[rng.integers(len(edges), size=600)].astype(float) * rng.choice([-1, 1], (600, 2))
    d[:30] = (5, 5)                                              # exactly at max_thr
    d[30:60] = (7, 2)                                            # just above it (53)
    x1, x2, models = _offsets_case(rng, d, p)
    _check(gpu_ctx, 1, x1, x2, models, 50.0 * 2.0 ** (-2 * p), -2.0, seed=p)


@pytest.mark.parametrize("what", ["equal", "zero", "deep", "crowded"])
def test_ties(gpu_ctx, what):
    rng = np.random.default_rng(len(what))
    M = 5000 if what == "crowded" else 700
    d = np.tile([1.0, 0.0], (M, 1))
    if what == "zero":
        d[:] = 0
    elif what == "deep":
        d[:400] = (2.0 ** -25, 0)                                # 50 binades below the bound: clamped into bin 0
        d[400:] = rng.integers(-3, 4, (M - 400, 2))
    elif what == "crowded":
        d[:4500] = (6, 0)                                        # thousands of residuals in one bin
        d[4500:] = rng.integers(-8, 9, (M - 4500, 2))
    x1, x2, models = _offsets_case(rng, d, 12, n_models=7)
    _check(gpu_ctx, 1, x1, x2, models, 64.0 * 2.0 ** -24, -1.5, seed=M)


# ---- the device and host evaluations of detmath agree bit for bit ------------------------------------------------
def test_detmath_device_equals_host(r3dlib, gpu_ctx):
    rng = np.random.default_rng(3)
    seams = np.ldexp(1.0, np.arange(-60, 61)).repeat(2) * np.tile([1.0, math.sqrt(0.5)], 121)
    ulps = np.arange(-2000, 2001)
    near = np.concatenate([s + ulps * np.spacing(s) for s in seams])
    cases = {
        r3dlib.DETMATH_LOG10: np.r_[near, 10.0 ** rng.uniform(-300, 300, 300000), rng.uniform(0, 2, 100000)],
        # the seven-point cubic: cube roots of |R| + sqrt(R^2 - Q^3) over many decades, cos of theta / 3 and
        # (theta +- 2 pi) / 3, acos of R / sqrt(Q^3) in [-1, 1]
        r3dlib.DETMATH_CBRT: np.r_[0.0, 10.0 ** rng.uniform(-200, 200, 400000), rng.uniform(0, 10, 100000)],
        r3dlib.DETMATH_COS: np.r_[rng.uniform(-math.pi, math.pi, 300000), rng.uniform(-2.1, 2.1, 100000),
                                  np.linspace(-math.pi, math.pi, 100001)],
        r3dlib.DETMATH_ACOS: np.r_[rng.uniform(-1, 1, 300000), 1 - 10.0 ** -rng.uniform(0, 16, 50000),
                                   -1 + 10.0 ** -rng.uniform(0, 16, 50000), -1.0, 1.0, 0.0],
    }
    total = 0
    for fn, x in cases.items():
        d = r3dlib.debug_detmath(fn, x, on_device=True)
        h = r3dlib.debug_detmath(fn, x, on_device=False)
        same = (d.view(np.uint64) == h.view(np.uint64)) | (np.isnan(d) & np.isnan(h))
        assert same.all(), "fn %d: device and host differ at x = %r (%r vs %r)" % (fn, x[~same][0], d[~same][0], h[~same][0])
        total += len(x)
    assert total >= 10 ** 6


# ---- end to end: the selected model, its inliers and errorMax from the returned model alone -----------------------
def _check_selection(model, res, inliers, n_inliers, found_precision, max_thr, M, logalpha0, delta):
    """inliers: indices in residual order; res: float64 residuals recomputed from the returned model.  delta: the
    absolute error of a recomputed point-to-point / point-to-line distance that comes from rebuilding the kernel's model
    from the returned pose or E (a few dozen ulp of the largest pixel coordinate)."""
    assert len(inliers) == n_inliers and len(set(inliers.tolist())) == n_inliers
    ins = res[inliers]
    rest = np.delete(res, inliers)
    emax = ins.max()
    assert emax <= max_thr * (1 + 1e-12)
    if len(rest):  # the k smallest (ties at the boundary rounded either way)
        assert emax <= np.nanmin(np.r_[rest, np.inf]) * (1 + 1e-9) + 1e-300
    tol = 1e-12 * emax + 2 * math.sqrt(emax) * delta + delta * delta
    assert abs(found_precision ** 2 - emax) <= tol, (found_precision ** 2, emax, tol)
    curve = ref.nfa_curve(model, res, M, max_thr, logalpha0)
    best, kbest = ref.best_nfa(curve)
    assert best < 0
    tol = 1e-6 * (1 + abs(best))
    assert kbest == n_inliers or curve.get(int(n_inliers), np.inf) <= best + tol, (kbest, n_inliers)


def _relpose_case(ctx, r3dlib, xI, xJ, K, precision):
    put = r3dlib.Matches.from_csr(np.array([[0, 1]], np.uint32), np.array([0, len(xI)], np.uint64),
                                  np.array(list(zip(range(len(xI)), range(len(xI)))), r3dlib.indmatch_dtype))
    ctx.clear_regions()
    ctx.upload_regions(0, np.zeros((len(xI), 16), np.float32), xI)
    ctx.upload_regions(1, np.zeros((len(xJ), 16), np.float32), xJ)
    got, inl = ctx.relative_poses(put, [W, W], [H, H], np.array([K, K]), precision_px=precision, refine=False)
    return got[0], inl.to_dict().get((0, 1))


@pytest.mark.parametrize("kind,precision", [("outliers60", 4.0), ("rotation", 4.0), ("large", 4.0), ("small", 4.0),
                                            ("outliers60", 0.05), ("outliers60", np.inf), ("small", np.inf)])
def test_relpose_selection(gpu_ctx, r3dlib, kind, precision):
    cases = []
    if kind == "outliers60":
        cases = [two_view(600, 1, outlier_frac=0.6)]
    elif kind == "rotation":
        cases = [two_view(500, 2, baseline=(1e-4, 0.0, 0.0), noise_px=0.3)]
    elif kind == "large":
        cases = [two_view(17000, 3, outlier_frac=0.3)]
    else:
        cases = [two_view(n, 20 + n, noise_px=0.2) for n in range(13, 21)]
    # every scene holds a clear majority of true matches: each pair must come back with a model, and each is checked
    unchecked = []
    for c, (xI, xJ, _, _, K) in enumerate(cases):
        g, inl = _relpose_case(gpu_ctx, r3dlib, xI, xJ, K, precision)
        if g["status"] != r3dlib.RELPOSE_OK or inl is None:
            unchecked.append((c, len(xI), int(g["status"])))
            continue
        F = _F_from_E(g["E"], K, K)
        res = ref.float_residuals(2, F.ravel(), xI.astype(np.float64), xJ.astype(np.float64))
        _check_selection(2, res, inl["i"].astype(np.int64), int(g["n_inliers"]), float(g["found_residual_precision"]),
                         precision ** 2, len(xI), _logalpha0(2, W, H), 64 * math.ulp(float(np.abs(xJ).max())))
    assert not unchecked, "pairs without a model (case, matches, status): %s" % unchecked


@pytest.mark.parametrize("kind,precision", [("outliers60", np.inf), ("large", np.inf), ("small", np.inf),
                                            ("outliers60", 0.05), ("small", 4.0)])
def test_resection_selection(gpu_ctx, r3dlib, kind, precision):
    if kind == "outliers60":
        views = [make_view(1, 600, model=1, outliers=0.6)]
    elif kind == "large":
        views = [make_view(2, 17000, model=1, outliers=0.3)]
    else:
        views = [make_view(30 + n, n, model=1, noise=0.2) for n in range(13, 21)]
    counts = [len(v["X"]) for v in views]
    rv = r3dlib.resection_views(counts, [v["width"] for v in views], [v["height"] for v in views], [1] * len(views),
                                [v["focal"] for v in views], [v["ppx"] for v in views], [v["ppy"] for v in views],
                                [v["disto"] for v in views])
    got, ofs, inl = gpu_ctx.resect_views(rv, np.concatenate([v["X"] for v in views]), np.concatenate([v["x"] for v in views]),
                                         precision_px=precision, refine=False)
    unchecked = [(a, len(v["X"]), int(g["status"])) for a, (g, v) in enumerate(zip(got, views)) if g["status"] != r3dlib.RESECT_OK]
    assert not unchecked, "views without a pose (view, correspondences, status): %s" % unchecked
    for a, (g, v) in enumerate(zip(got, views)):
        Kt = np.array([[v["focal"], 0, v["ppx"]], [0, v["focal"], v["ppy"]], [0, 0, 1.0]])
        P = Kt @ np.c_[g["rotation_ransac"], g["translation_ransac"]]
        res = ref.float_residuals(3, P.ravel(), v["X"][:, :2], v["x"], v["X"][:, 2])
        _check_selection(3, res, inl[int(ofs[a]):int(ofs[a + 1])].astype(np.int64), int(g["n_inliers"]),
                         float(g["found_residual_precision"]), precision ** 2, len(v["X"]),
                         _logalpha0(3, v["width"], v["height"]), 64 * math.ulp(float(np.abs(v["x"]).max())))
