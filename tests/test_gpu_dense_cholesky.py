"""-m gpu: the dense linear-algebra core shared by bundle adjustment, rotation averaging and translation averaging --
k_chol_fused, k_chol_envelope and k_rotavg_trsm3 -- run on matrices built here, through r3d_debug_cholesky and
r3d_debug_chol_solve3 (the launch code the solvers use), against plain references:

  exact      unit lower-triangular L with entries in {-1, 0, 1}, A = L L^T, b = A x* (x* small integers).  Every
             partial sum either kernel forms is an integer below 2^50 (checked here, with integer arithmetic, before the
             kernel runs), so every operation is exact and L, y = L^T x*, x* and the block inverses must come back
             bit for bit.  This rests on rsqrt(1.0) == 1.0 on the device, which the first test pins.
  float64    A = Q diag(lambda) Q^T or a banded + bordered SPD matrix shaped like BA's reduced camera system:
             ||A - L L^T||_F <= c n u ||A||_F, ||A x - b|| <= c n u ||A|| ||x||, ||x - x_scipy|| <= c n u kappa ||x||.
  bits       the upper triangle is never read, the grid / cluster size does not change a bit, repeated calls agree.
  flag       the not-positive-definite flag the three LM loops reject a step on.

Sizes cover partial and full panels, the rhs row inside the last diagonal tile and in a tile of its own, the
grid-stride loops of k_chol_fused (n >= 4257: more row tiles than the 132 CTAs of one per SM) and k_rotavg_trsm3
(n > 2144), and R3D_ROTAVG_MAX_VIEWS * 3 = 12288."""
import functools

import numpy as np
import pytest
import scipy.linalg
import scipy.sparse as sp
import scipy.sparse.linalg

from regard3d_b200 import capi

pytestmark = pytest.mark.gpu

NB = 32
U = 2.0 ** -53
C_BAR = 8.0                 # the constant of the float64 bars
EXACT_LIMIT = 2 ** 50       # partial sums of the exact fixtures stay below this
ENV_MAX_ACTIVE = 24         # kEnvMaxActive (ba.cu)
DENSE, ENV = capi.CHOL_DENSE, capi.CHOL_ENVELOPE
ERR_INVALID = -1

EXACT_SIZES = [1, 2, 3, 31, 32, 33, 63, 64, 65, 96, 97, 177, 228, 288, 1206, 2145, 4255, 4256, 4257, 12288]


# ---- fixtures ------------------------------------------------------------------------------------------------------
def int_factor(n, seed, band=8, border=None, reach0_tiles=(), wrap=0, density=0.5):
    """Unit lower-triangular L (CSR, int64), entries in {-1, 0, 1}: `band` sub-diagonals; the last `border` rows dense
    from column 0 (BA's intrinsics rows); rows of `reach0_tiles` dense from column 0; the `wrap` camera rows before the
    border reaching back to columns 0..band-1 (a closed image sequence).  Returns (L, first column of every row)."""
    rng = np.random.default_rng(seed)
    if border is None:
        border = min(6, n // 5)
    ii, jj = [np.arange(n)], [np.arange(n)]
    for d in range(1, band + 1):                         # the band
        i = np.arange(d, n)
        ii.append(i)
        jj.append(i - d)
    long_rows = set(range(n - border, n))
    for t in reach0_tiles:
        long_rows.update(range(t * NB, min((t + 1) * NB, n - border)))
    for i in sorted(long_rows):                          # dense left of the band
        j = np.arange(0, max(i - band, 0))
        ii.append(np.full(len(j), i))
        jj.append(j)
    for i in range(max(n - border - wrap, 0), n - border):
        if i not in long_rows:
            j = np.arange(0, max(min(band, i - band), 0))
            ii.append(np.full(len(j), i))
            jj.append(j)
    i, j = np.concatenate(ii), np.concatenate(jj)
    off = i != j
    v = np.ones(len(i), np.int64)
    v[off] = rng.choice([-1, 1], off.sum()) * (rng.random(off.sum()) < density)
    L = sp.csr_matrix((v, (i, j)), shape=(n, n), dtype=np.int64)
    L.eliminate_zeros()
    first = np.arange(n)
    coo = L.tocoo()
    np.minimum.at(first, coo.row, coo.col)
    return L, first


def ft_of(first, n):
    """First column tile of every row tile (rows 0..n, row n = the rhs, which reaches column 0)."""
    first = np.append(first, 0)
    ntr = (n + 1 + NB - 1) // NB
    return np.array([first[t * NB:min((t + 1) * NB, n + 1)].min() // NB for t in range(ntr)], np.int32)


def max_active(ft, n):
    nblk, ntr = (n + NB - 1) // NB, (n + 1 + NB - 1) // NB
    return max(int(np.sum(ft[k + 1:ntr] <= k)) for k in range(nblk))


def diag_blocks(L, n, absolute=False):
    """The 32 x 32 diagonal blocks of L (identity-padded) and their exact integer inverses, or with absolute=True the
    inverses of the comparison matrices (2I - |L_kk|): nonnegative bounds of every intermediate of a substitution."""
    nblk = (n + NB - 1) // NB
    D = np.zeros((nblk, NB, NB), np.int64)
    D[:, np.arange(NB), np.arange(NB)] = 1
    coo = L.tocoo()
    m = coo.row // NB == coo.col // NB
    D[coo.row[m] // NB, coo.row[m] % NB, coo.col[m] % NB] = np.abs(coo.data[m]) if absolute else coo.data[m]
    M = np.zeros_like(D)
    for r in range(NB):
        s = np.einsum("bj,bjc->bc", D[:, r, :r], M[:, :r, :])
        M[:, r, :] = -s if not absolute else s
        M[:, r, r] += 1
    return D, M


def blockdiag(M, n):
    nblk = M.shape[0]
    return sp.block_diag([sp.csr_matrix(M[k]) for k in range(nblk)], format="csr", dtype=np.int64)[:n, :n]


def exact_bound(L, y, xs):
    """Largest magnitude of any partial sum the kernels form on A = L L^T, b = L y (y = L^T xs): Schur complements
    and syrk sums (|L'| |L'|^T with L' = [L; y^T], twice for the envelope's substitution), the dense kernel's block
    products A_panel Linv_k^T, and the backward substitutions.  Integer arithmetic throughout."""
    n = L.shape[0]
    Lp = sp.vstack([abs(L), sp.csr_matrix(np.abs(y)[None, :])]).tocsr().astype(np.int64)
    S1 = (Lp @ Lp.T).tocsr()
    _, Mabs = diag_blocks(L, n, absolute=True)
    Mb = blockdiag(Mabs, n)
    trsm = S1[:, :n] @ Mb.T
    zb = np.abs(y) + abs(L).T @ np.abs(xs)
    back = Mb.T @ zb
    return max(2 * int(S1.max()), int(trsm.max()), int(back.max()), 2 * int(zb.max()))


@functools.lru_cache(maxsize=1)
def exact_fixture(n, seed=1):
    """Sparse parts only (the dense A is built per test, so no 1.2 GB matrix outlives its test)."""
    L, first = int_factor(n, seed)
    xs = np.random.default_rng(seed + 1).integers(-3, 4, n).astype(np.int64)
    y = L.T @ xs
    b = L @ y
    bound = exact_bound(L, y, xs)
    assert bound < EXACT_LIMIT, bound
    return L, first, xs, y, b


def dense_A(L, b):
    """(n+1) x n float64: L L^T (from the sparse product, never a dense one) and b as row n."""
    n = L.shape[0]
    A = np.zeros((n + 1, n))
    P = (L @ L.T).tocoo()
    A[P.row, P.col] = P.data
    A[n] = b
    return A


def check_exact(L_out, x_out, L, y, xs):
    n = L.shape[0]
    coo = L.tocoo()
    assert np.array_equal(L_out[coo.row, coo.col], coo.data.astype(np.float64)), "factor entries"
    assert np.count_nonzero(L_out[:n]) == L.nnz, "non-zeros outside the pattern of L (or above the diagonal)"
    assert np.array_equal(L_out[n], y.astype(np.float64)), "forward substitution y = L^-1 b"
    assert np.array_equal(x_out, xs.astype(np.float64)), "solution"


def spd_spectrum(n, kappa, seed):
    """A = Q diag(lambda) Q^T, lambda geometric from 1 down to 1/kappa."""
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    lam = np.logspace(0, -np.log10(kappa), n)
    A = (Q * lam) @ Q.T
    return 0.5 * (A + A.T), 1.0, float(kappa)


def ba_like(n, seed, scale_decades=0.0, band=14, border=6):
    """A banded + bordered SPD matrix shaped like BA's reduced camera system: B B^T + I with B lower band + dense
    border rows, then D A D with log10 D uniform in +-scale_decades (the conditioning).  Returns (A, first column of
    every row, ||A||_2, kappa)."""
    rng = np.random.default_rng(seed)
    i, j = [], []
    for d in range(0, band + 1):
        r = np.arange(d, n - border)
        i.append(r)
        j.append(r - d)
    for r in range(n - border, n):
        i.append(np.full(r + 1, r))
        j.append(np.arange(r + 1))
    i, j = np.concatenate(i), np.concatenate(j)
    B = sp.csr_matrix((rng.standard_normal(len(i)), (i, j)), shape=(n, n))
    A = (B @ B.T).toarray() + np.eye(n)
    d = 10.0 ** rng.uniform(-scale_decades, scale_decades, n)
    A = d[:, None] * A * d[None, :]
    A = 0.5 * (A + A.T)
    ev = np.linalg.eigvalsh(A)
    first = np.maximum(np.arange(n) - band, 0)
    first[n - border:] = 0
    return A, first, float(ev[-1]), float(ev[-1] / ev[0])


def with_rhs(A, b):
    return np.vstack([A, b[None, :]])


def check_float_bars(A, b, L_out, x, normA, kappa, x_ref):
    n = A.shape[0]
    L = np.tril(L_out[:n])
    assert np.array_equal(L_out[:n], L), "entries above the diagonal"
    assert np.linalg.norm(A - L @ L.T) <= C_BAR * n * U * np.linalg.norm(A)
    assert np.linalg.norm(A @ x - b) <= C_BAR * n * U * normA * np.linalg.norm(x)
    assert np.linalg.norm(x - x_ref) <= C_BAR * n * U * kappa * np.linalg.norm(x)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


# ---- a. exact integer fixtures -------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", [DENSE, ENV])
def test_identity_factors_to_itself(gpu_ctx, method):
    """rsqrt(1.0) == 1.0 on the device: the premise of every bit-exact bar below."""
    n = 64
    A = np.vstack([np.eye(n), np.arange(n, dtype=np.float64)[None, :]])
    ft = np.append(np.arange((n + NB) // NB - 1), 0).astype(np.int32)
    L, x, Linv, bad = gpu_ctx.debug_cholesky(A, method, ft=ft if method == ENV else None)
    assert not bad
    assert np.array_equal(L[:n], np.eye(n)) and np.array_equal(L[n], A[n]) and np.array_equal(x, A[n])
    if method == DENSE:
        assert np.array_equal(Linv, np.broadcast_to(np.eye(NB), Linv.shape))


@pytest.mark.parametrize("n,method", [(n, m) for n in EXACT_SIZES for m in (DENSE, ENV) if m == DENSE or n % 2 == 0])
def test_exact(gpu_ctx, n, method):
    """Dense kernel at every size, envelope kernel (even n only) with ft from the fixture's tile profile."""
    L, first, xs, y, b = exact_fixture(n)
    A = dense_A(L, b)
    ft = ft_of(first, n)
    if method == ENV:
        assert max_active(ft, n) <= ENV_MAX_ACTIVE
    L_out, x_out, Linv, bad = gpu_ctx.debug_cholesky(A, method, ft=ft if method == ENV else None)
    assert not bad
    check_exact(L_out, x_out, L, y, xs)
    if method == DENSE:
        _, M = diag_blocks(L, n)
        assert np.array_equal(Linv, M.astype(np.float64)), "inverses of the diagonal blocks"


# ---- b. float64 SPD matrices with controlled conditioning ----------------------------------------------------------
@pytest.mark.parametrize("n", [64, 300, 1206])
@pytest.mark.parametrize("kappa", [1e2, 1e8, 1e12])
def test_dense_spectrum_bars(gpu_ctx, n, kappa):
    A, normA, kappa = spd_spectrum(n, kappa, seed=n)
    b = A @ np.random.default_rng(7).standard_normal(n)
    L_out, x, _, bad = gpu_ctx.debug_cholesky(with_rhs(A, b), DENSE)
    assert not bad
    check_float_bars(A, b, L_out, x, normA, kappa, scipy.linalg.cho_solve(scipy.linalg.cho_factor(A, lower=True), b))


@pytest.mark.parametrize("n", [228, 288, 1206])
@pytest.mark.parametrize("decades", [0.0, 1.5, 2.5])
def test_ba_like_both_kernels_bars(gpu_ctx, n, decades):
    A, first, normA, kappa = ba_like(n, seed=n + int(2 * decades), scale_decades=decades)
    b = A @ np.random.default_rng(9).standard_normal(n)
    x_ref = scipy.linalg.cho_solve(scipy.linalg.cho_factor(A, lower=True), b)
    Ab = with_rhs(A, b)
    Ld, xd, _, bad_d = gpu_ctx.debug_cholesky(Ab, DENSE)
    Le, xe, _, bad_e = gpu_ctx.debug_cholesky(Ab, ENV, ft=ft_of(first, n))
    assert not bad_d and not bad_e
    check_float_bars(A, b, Ld, xd, normA, kappa, x_ref)
    check_float_bars(A, b, Le, xe, normA, kappa, x_ref)
    assert np.linalg.norm(xe - xd) <= 2 * C_BAR * n * U * kappa * np.linalg.norm(xd)
    assert np.linalg.norm(Le - Ld) <= 2 * C_BAR * n * U * kappa * np.linalg.norm(Ld)


# ---- c. contracts and determinism ----------------------------------------------------------------------------------
def gram(n, seed, k=256):
    """A rounding-sensitive dense SPD matrix (every entry a sum of k products) with a random rhs row."""
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n, k))
    A = G @ G.T / k + 0.05 * np.eye(n)
    return with_rhs(A, rng.standard_normal(n))


@pytest.mark.parametrize("n", [228, 288])
@pytest.mark.parametrize("method", [DENSE, ENV])
def test_upper_triangle_is_not_read(gpu_ctx, n, method):
    A, first, _, _ = ba_like(n, seed=3, scale_decades=1.0)
    Ab = with_rhs(A, np.random.default_rng(4).standard_normal(n))
    An = Ab.copy()
    An[np.triu_indices(n, 1)] = np.nan
    ft = ft_of(first, n) if method == ENV else None
    ref = gpu_ctx.debug_cholesky(Ab, method, ft=ft)
    got = gpu_ctx.debug_cholesky(An, method, ft=ft)
    assert not ref[3] and not got[3]
    for r, g in zip(ref[:3], got[:3]):
        if r is not None:
            assert np.array_equal(bits(r), bits(g))


@pytest.mark.parametrize("n", [300, 4257])
def test_dense_bits_do_not_depend_on_the_grid(gpu_ctx, n):
    """Grid 1 drives every grid-stride loop of k_chol_fused at any n; one writer per tile, fixed reduction order."""
    Ab = gram(n, seed=n)
    ref = gpu_ctx.debug_cholesky(Ab, DENSE, grid=0)
    again = gpu_ctx.debug_cholesky(Ab, DENSE, grid=0)
    for grid, got in [(0, again)] + [(g, gpu_ctx.debug_cholesky(Ab, DENSE, grid=g)) for g in (1, 2, 5)]:
        assert not got[3]
        for r, g in zip(ref[:3], got[:3]):
            assert np.array_equal(bits(r), bits(g)), "grid %d" % grid


@pytest.mark.parametrize("n", [228, 288])
def test_envelope_bits_do_not_depend_on_the_cluster(gpu_ctx, n):
    A, first, _, _ = ba_like(n, seed=5, scale_decades=2.0)
    Ab = with_rhs(A, np.random.default_rng(6).standard_normal(n))
    ft = ft_of(first, n)
    ref = gpu_ctx.debug_cholesky(Ab, ENV, ft=ft, grid=1)
    for ctas in list(range(1, 9)) + [0]:
        got = gpu_ctx.debug_cholesky(Ab, ENV, ft=ft, grid=ctas)
        assert not got[3]
        assert np.array_equal(bits(ref[0]), bits(got[0])) and np.array_equal(bits(ref[1]), bits(got[1])), "cluster %d" % ctas


@pytest.mark.parametrize("n", [300, 2145])
def test_trsm3_bits_do_not_depend_on_the_grid(gpu_ctx, n):
    A = gram(n, seed=n + 1)[:n]
    Y = np.random.default_rng(n).standard_normal((n, 3))
    ref = gpu_ctx.debug_chol_solve3(A, Y, grid=0)
    for grid in (0, 1, 3):
        assert np.array_equal(bits(ref), bits(gpu_ctx.debug_chol_solve3(A, Y, grid=grid))), "grid %d" % grid


# ---- d. the not-positive-definite flag -----------------------------------------------------------------------------
FLAG_N = 80  # 2.5 panels: index 70 lies in the partial last one


def flag_matrix(kind, p, n=FLAG_N):
    """Exact integer A (every pivot before p is exactly 1) whose factorisation meets at index p: a pivot of -1
    ("negative"), an exact 0 (row and column p duplicate row and column p - 5), or a NaN below the diagonal."""
    L, first = int_factor(n, seed=11, band=6, border=0)
    d = np.ones(n)
    if kind == "negative":
        d[p] = -1.0
    Ld = L.toarray().astype(np.float64)
    A = (Ld * d) @ Ld.T
    if kind == "zero":
        q = p - 5
        A[p, :], A[:, p] = A[q, :], A[:, q]
        A[p, p] = A[q, q]
    if kind == "nan":
        A[p, p - 3] = np.nan
    return with_rhs(A, np.ones(n)), ft_of(np.maximum(np.arange(n) - 8, 0), n)


@pytest.mark.parametrize("method", [DENSE, ENV])
@pytest.mark.parametrize("kind,p", [("negative", 0), ("negative", 31), ("negative", 32), ("negative", 70),
                                    ("zero", 31), ("zero", 70), ("nan", 40), ("nan", 70)])
def test_not_positive_definite_sets_the_flag(gpu_ctx, method, kind, p):
    Ab, ft = flag_matrix(kind, p)
    assert gpu_ctx.debug_cholesky(Ab, method, ft=ft if method == ENV else None)[3]


@pytest.mark.parametrize("method", [DENSE, ENV])
def test_ill_conditioned_positive_definite_leaves_the_flag_clear(gpu_ctx, method):
    n = FLAG_N
    A, normA, _ = spd_spectrum(n, 1e12, seed=12)
    Lnp = np.linalg.cholesky(A)
    assert np.diag(Lnp).min() ** 2 > 50 * n * U * normA  # the smallest pivot is far above rounding
    ft = np.zeros((n + NB) // NB, np.int32)
    Ab = with_rhs(A, np.ones(n))
    bad, _ = flag_matrix("negative", 31)
    assert gpu_ctx.debug_cholesky(bad, method, ft=ft)[3]
    assert not gpu_ctx.debug_cholesky(Ab, method, ft=ft if method == ENV else None)[3]  # and the hook clears the flag


# ---- e. envelope profiles ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [96, 228, 288, 1206])
def test_envelope_wrap_around(gpu_ctx, n):
    """A closed image sequence: the last camera rows reach back to column 0."""
    L, first = int_factor(n, seed=21, wrap=40)
    xs = np.random.default_rng(22).integers(-3, 4, n)
    y = L.T @ xs
    assert exact_bound(L, y, xs) < EXACT_LIMIT
    ft = ft_of(first, n)
    assert ft[(n - 8) // NB] == 0 and max_active(ft, n) <= ENV_MAX_ACTIVE
    L_out, x_out, _, bad = gpu_ctx.debug_cholesky(dense_A(L, L @ y), ENV, ft=ft)
    assert not bad
    check_exact(L_out, x_out, L, y, xs)


def profile_with_active(n_active):
    """n = 1280 (rhs row in a tile of its own); tiles 2 .. reach column 0, so panel 0 has n_active active row tiles
    (tile 1 through the band, the border tile 39, the rhs tile 40)."""
    n = 1280
    L, first = int_factor(n, seed=31, band=6, reach0_tiles=range(2, 2 + n_active - 3), density=0.3)
    return n, L, first


def test_envelope_24_active_row_tiles(gpu_ctx):
    n, L, first = profile_with_active(ENV_MAX_ACTIVE)
    ft = ft_of(first, n)
    assert max_active(ft, n) == ENV_MAX_ACTIVE
    xs = np.random.default_rng(32).integers(-3, 4, n)
    y = L.T @ xs
    assert exact_bound(L, y, xs) < EXACT_LIMIT
    L_out, x_out, _, bad = gpu_ctx.debug_cholesky(dense_A(L, L @ y), ENV, ft=ft)
    assert not bad
    check_exact(L_out, x_out, L, y, xs)


def test_bad_arguments_are_rejected_on_the_host(gpu_ctx):
    n, L, first = profile_with_active(ENV_MAX_ACTIVE + 1)
    ft = ft_of(first, n)
    assert max_active(ft, n) == ENV_MAX_ACTIVE + 1
    A = dense_A(L, np.zeros(n))

    def rejected(f, *a, **k):
        with pytest.raises(capi.R3DError) as e:
            f(*a, **k)
        return e.value.code == ERR_INVALID

    assert rejected(gpu_ctx.debug_cholesky, A, ENV, ft=ft)                       # 25 active row tiles
    small = with_rhs(np.eye(64), np.ones(64))
    ft64 = np.array([0, 1, 0], np.int32)
    assert rejected(gpu_ctx.debug_cholesky, np.zeros((1, 0)), DENSE)             # n < 1
    assert rejected(gpu_ctx.debug_cholesky, with_rhs(np.eye(63), np.ones(63)), ENV, ft=np.zeros(2, np.int32))  # odd n
    assert rejected(gpu_ctx.debug_cholesky, small, ENV, ft=np.array([0, 2, 0], np.int32))   # ft[t] > t
    assert rejected(gpu_ctx.debug_cholesky, small, ENV, ft=np.array([0, -1, 0], np.int32))
    assert rejected(gpu_ctx.debug_cholesky, small, ENV, ft=None)
    assert rejected(gpu_ctx.debug_cholesky, small, ENV, ft=ft64, grid=9)         # cluster > 8
    assert rejected(gpu_ctx.debug_cholesky, small, DENSE, grid=100000)           # more CTAs than can be co-resident
    assert rejected(gpu_ctx.debug_cholesky, small, DENSE, grid=-1)
    assert rejected(gpu_ctx.debug_chol_solve3, np.eye(64), np.ones((64, 3)), grid=100000)
    for short in (ft64[:2], np.zeros(4, np.int32)):                                # one entry per row tile, no more
        with pytest.raises(ValueError):
            gpu_ctx.debug_cholesky(small, ENV, ft=short)
    assert not gpu_ctx.debug_cholesky(small, ENV, ft=ft64, grid=8)[3]           # and the context still works


# ---- f. k_rotavg_trsm3 ---------------------------------------------------------------------------------------------
def trsm3_bound(L, Xs):
    """Largest partial sum of the factorisation of A = L L^T and of the two blocked substitutions on Y = A Xs."""
    n = L.shape[0]
    zb = abs(L).T @ np.abs(Xs)          # >= |L^T Xs| and every backward partial sum
    Yb = abs(L) @ zb                    # >= |Y| and every forward partial sum (twice)
    _, Mabs = diag_blocks(L, n, absolute=True)
    Mb = blockdiag(Mabs, n)
    zero = np.zeros(n, np.int64)        # the factorisation, its rhs row zero
    return max(exact_bound(L, zero, zero), 2 * int(Yb.max()), int((Mb @ Yb).max()), 2 * int((Mb.T @ zb).max()))


@pytest.mark.parametrize("n", [1, 33, 64, 97, 300, 2145, 4257, 12288])
def test_trsm3_exact(gpu_ctx, n):
    L, _ = int_factor(n, seed=41)
    Xs = np.random.default_rng(42).integers(-3, 4, (n, 3)).astype(np.int64)
    assert trsm3_bound(L, Xs) < EXACT_LIMIT
    Y = (L @ (L.T @ Xs)).astype(np.float64)
    A = dense_A(L, np.zeros(n))[:n]
    assert np.array_equal(gpu_ctx.debug_chol_solve3(A, Y), Xs.astype(np.float64))


@pytest.mark.parametrize("n", [300, 1206])
def test_trsm3_against_cho_solve(gpu_ctx, n):
    A, normA, kappa = spd_spectrum(n, 1e8, seed=n + 2)
    Y = np.random.default_rng(n).standard_normal((n, 3))
    X = gpu_ctx.debug_chol_solve3(A, Y)
    X_ref = scipy.linalg.cho_solve(scipy.linalg.cho_factor(A, lower=True), Y)
    for c in range(3):
        assert np.linalg.norm(A @ X[:, c] - Y[:, c]) <= C_BAR * n * U * normA * np.linalg.norm(X[:, c])
        assert np.linalg.norm(X[:, c] - X_ref[:, c]) <= C_BAR * n * U * kappa * np.linalg.norm(X[:, c])


@pytest.mark.parametrize("n", [2145, 4257, 12288])
def test_trsm3_residual_large(gpu_ctx, n):
    """Random right-hand sides on banded + bordered float SPD systems, residual bar (no dense reference at this size)."""
    rng = np.random.default_rng(n)
    band, border = 14, 6
    i, j = [], []
    for d in range(band + 1):
        r = np.arange(d, n - border)
        i.append(r)
        j.append(r - d)
    for r in range(n - border, n):
        i.append(np.full(r + 1, r))
        j.append(np.arange(r + 1))
    i, j = np.concatenate(i), np.concatenate(j)
    B = sp.csr_matrix((rng.standard_normal(len(i)), (i, j)), shape=(n, n))
    As = (B @ B.T + sp.identity(n)).tocsr()
    A = np.zeros((n, n))
    P = As.tocoo()
    A[P.row, P.col] = P.data
    normA = float(scipy.sparse.linalg.eigsh(As, k=1, which="LA", return_eigenvectors=False)[0])
    Y = rng.standard_normal((n, 3))
    X = gpu_ctx.debug_chol_solve3(A, Y)
    R = As @ X - Y
    for c in range(3):
        assert np.linalg.norm(R[:, c]) <= C_BAR * n * U * normA * np.linalg.norm(X[:, c])
