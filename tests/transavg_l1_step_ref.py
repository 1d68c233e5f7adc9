"""Reference of one interior-point iteration of r3d_translation_averaging_l1 (what r3d_debug_transavg_l1_step returns),
built from the linear program itself rather than from the library's per-edge formulas.

The LP on the kept edges, in the library's variable order: x = (T of the free kept views, lambda per kept edge, gamma),
y = (T, gamma); per edge 7 rows of G x + s = h, s >= 0 (r_k - gamma, -r_k - gamma for k = 0..2, -lambda; r = T_J -
R_IJ T_I - lambda u_IJ), c = e_gamma.  One iteration at (x, s, z) is Mehrotra's: D = Z S^-1, the Newton system
G^T D G dx = -(c + G^T (z + wt)), wt = (z rp - rc) / s, rp = G x + s - h, with lambda eliminated by its Schur complement;
the reduced (T, gamma) system scaled to a unit diagonal; ds = -rp - G dx, dz = wt + D G dx; the ratio test with eta = 1
(predictor) and 0.99 (corrector); sigma = (mu_aff / mu)^3.

Two precisions:
  exact()    fractions.Fraction on the float64 inputs (small scenes): the assembled reduced matrix and right-hand side,
             the norms, and the exact solution of the scaled system the library factored.
  Step       float64, every value with a magnitude A: the same sum taken over the absolute values of its terms, as in
             ba_step_ref.py.  A kernel that is right to round-off lands within a small multiple of u A; one that drops
             or misplaces a term does not.
check() holds a library step (or emulate()'s stand-in for one) to a Step and returns the worst ratios per quantity.
"""
import math
from fractions import Fraction

import numpy as np
import scipy.sparse as sp

U = np.finfo(np.float64).eps / 2
ROWS = 7
ETA = 0.99
REG_REL = 1e-18
REG_GROWTH = 100.0
REG_TRIES = 5
MUTANTS = ("gamma_schur", "c_gamma", "swap_reversed", "corrector_wt", "sz_edge")


class Scene:
    """The kept edges as the kernels see them: m views, per edge the record-oriented local (I, J), R_IJ and u_IJ."""

    def __init__(self, m, edge_ij, Rij, u, edge_record=None):
        self.m = int(m)
        self.ij = np.asarray(edge_ij, np.int64).reshape(-1, 2)
        self.R = np.asarray(Rij, np.float64).reshape(-1, 3, 3)
        self.u = np.asarray(u, np.float64).reshape(-1, 3)
        self.record = edge_record
        self.ne = len(self.ij)
        self.nt = 3 * (self.m - 1)
        self.N = self.nt + 1
        self.nv = self.nt + self.ne + 1
        self.nr = ROWS * self.ne

    @classmethod
    def from_device(cls, D):
        return cls(D["m"], D["edge_ij"], D["Rij"], D["u"], D["edge_record"])

    def rows(self, swap_reversed=False):
        """G as a list of rows, each a list of (column, value), values as stored (float)."""
        out = []
        for e in range(self.ne):
            I, J = self.ij[e]
            R = self.R[e]
            if swap_reversed and I > J:  # a mutant: the canonical (lo, hi) in place of the record's orientation
                I, J = J, I
            lam = self.nt + e
            for sign in (1.0, -1.0):
                for k in range(3):
                    t = []
                    if J > 0:
                        t.append((3 * (J - 1) + k, sign))
                    if I > 0:
                        t += [(3 * (I - 1) + c, -sign * R[k, c]) for c in range(3)]
                    t += [(lam, -sign * self.u[e, k]), (self.nv - 1, -1.0)]
                    out.append(t)
            out.append([(lam, -1.0)])
        return out

    def G(self, swap_reversed=False):
        r, c, v = [], [], []
        for i, row in enumerate(self.rows(swap_reversed)):
            for j, x in row:
                r.append(i); c.append(j); v.append(x)
        return sp.csr_matrix((v, (r, c)), shape=(self.nr, self.nv))

    def h(self):
        h = np.zeros(self.nr)
        h[6::7] = -1.0
        return h

    def c(self):
        c = np.zeros(self.nv)
        c[-1] = 1.0
        return c

    def full(self, y, lam):
        return np.concatenate([y[:-1], lam, y[-1:]])

    def xidx(self):
        return np.r_[np.arange(self.nt), self.nv - 1]

    def lidx(self):
        return np.arange(self.nt, self.nt + self.ne)


def start_state(sc):
    """The solver's start point: T = 0, lambda = 2, gamma = 3, s = h - G y in the library's order of operations, z = 1."""
    y = np.zeros(sc.N)
    y[-1] = 3.0
    lam = np.full(sc.ne, 2.0)
    s = np.empty(sc.nr)
    for e in range(sc.ne):
        r = (0.0 - 0.0) - lam[e] * sc.u[e]  # T_J - R T_I at T = 0 is exactly 0
        s[7 * e:7 * e + 3] = -(r - y[-1])
        s[7 * e + 3:7 * e + 6] = -(-r - y[-1])
        s[7 * e + 6] = -(-lam[e] + 1.0)
    return y, lam, s, np.ones(sc.nr)


def regularised(Ms, k):
    """The scaled system of the k-th retry as the library forms it: diag + (1e-18 * 100^(k-1)) * max diag, rounded."""
    if k == 0:
        return Ms
    reg = REG_REL
    for _ in range(k - 1):
        reg *= REG_GROWTH
    d = np.diagonal(Ms)
    out = Ms.copy()
    out[np.arange(len(d)), np.arange(len(d))] = d + reg * np.fmax.reduce(np.r_[0.0, d])
    return out


def scaled_system(A):
    """M_s = (A sc_i) sc_j and b = rhs sc as the library's k_tl_jacobi forms them from its unscaled (N + 1) x N output;
    the lower triangle mirrored (the factorisation reads only it)."""
    N = A.shape[1]
    d = np.diagonal(A[:N])
    sc = np.where(d > 0, 1.0 / np.sqrt(np.where(d > 0, d, 1.0)), 1.0)
    Ms = (A[:N] * sc[:, None]) * sc[None, :]
    Ms = np.tril(Ms) + np.tril(Ms, -1).T
    return Ms, A[N] * sc, sc


class Step:
    """The float64 reference at one state, with magnitudes.  mutate: names from MUTANTS, deliberately wrong variants
    for the tests of the bars."""

    def __init__(self, sc, y, lam, s, z, mutate=()):
        self.sc_, self.mut = sc, set(mutate)
        self.y, self.lam, self.s, self.z = (np.asarray(a, np.float64) for a in (y, lam, s, z))
        G = sc.G("swap_reversed" in self.mut)
        self.Gm, self.Gt, self.Gmt = G, G.T.tocsr(), abs(G).T.tocsr()
        self.Gabs = abs(G).tocsr()
        x = sc.full(self.y, self.lam)
        h, c = sc.h(), sc.c()
        self.h, self.c = h, c
        gx = G @ x
        self.A_gx = self.Gabs @ np.abs(x)
        self.rp = (gx - h) + self.s
        self.A_rp = self.A_gx + np.abs(h) + np.abs(self.s)
        self.viol_rows = gx - h
        self.rd, self.A_rd = self.dual_residual(np.zeros(sc.nr)), np.abs(c) + self.Gmt @ np.abs(self.z)
        self.d = self.z / self.s
        # M = G^T D G and its magnitude, then lambda eliminated
        Dm = sp.diags(self.d)
        M = (self.Gt @ Dm @ G).tocsc()
        Mm = (self.Gmt @ Dm @ self.Gabs).tocsc()
        xi, li = sc.xidx(), sc.lidx()
        self.V = M[li][:, li].diagonal()
        self.Mxl, self.Mxl_m = M[xi][:, li].tocsr(), Mm[xi][:, li].tocsr()
        schur = (self.Mxl @ sp.diags(1.0 / self.V) @ self.Mxl.T).toarray()
        schur_m = (self.Mxl_m @ sp.diags(1.0 / self.V) @ self.Mxl_m.T).toarray()
        if "gamma_schur" in self.mut:
            schur[-1, :] = 0.0
        self.Mred = M[xi][:, xi].toarray() - schur
        self.A_Mred = Mm[xi][:, xi].toarray() + schur_m

    def norms(self):
        """(values, magnitudes) of k_tl_norms' five outputs."""
        s, z = self.s, self.z
        sz = s * z
        if "sz_edge" in self.mut:
            sz = sz.copy()
            sz[:7] = 0.0
        zl = z[6::7]
        val = [np.abs(self.rp).max(), max(0.0, self.viol_rows.max()), np.abs(self.rd).max(), math.fsum(sz), math.fsum(zl)]
        A = [self.A_rp.max(), (self.A_gx + np.abs(self.h)).max(), self.A_rd.max(), math.fsum(np.abs(s * z)), math.fsum(np.abs(zl))]
        return np.array(val), np.array(A)

    def rhs(self, rc, A_rc, wt_rc=None):
        """The reduced right-hand side -(c + G^T (z + wt)) with lambda eliminated, its magnitude, and the full one.
        wt_rc: the complementarity term the corrector's wt is formed with (a mutant passes the predictor's)."""
        s, z, sc = self.s, self.z, self.sc_
        wt = (z * self.rp - (rc if wt_rc is None else wt_rc)) / s
        A_wt = (z * self.A_rp + A_rc) / s + np.abs(wt)
        v = z + wt
        c = self.c.copy()
        if "c_gamma" in self.mut:
            c[-1] = 0.0
        full = -(c + self.Gt @ v)
        A_full = np.abs(c) + self.Gmt @ (np.abs(z) + A_wt)
        xi, li = sc.xidx(), sc.lidx()
        rl, A_rl = full[li], A_full[li]
        red = full[xi] - self.Mxl @ (rl / self.V)
        A_red = A_full[xi] + self.Mxl_m @ (A_rl / self.V)
        return dict(wt=wt, A_wt=A_wt, full=full, A_full=A_full, red=red, A_red=A_red, rl=rl, A_rl=A_rl)

    def back(self, dy, dlam, R):
        """Given the library's dy and dlam: dlam, ds, dz and their magnitudes.  R: rhs()'s dict."""
        sc = self.sc_
        dX = np.asarray(dy, np.float64)
        xl = self.Mxl.T @ dX
        dl = (R["rl"] - xl) / self.V
        A_dl = (R["A_rl"] + self.Mxl_m.T @ np.abs(dX)) / self.V + np.abs(dl)
        dxf = sc.full(dX, dlam)
        gd = self.Gm @ dxf
        A_gd = self.Gabs @ np.abs(dxf)
        ds = -self.rp - gd
        dz = R["wt"] + self.d * gd
        return dict(dlam=dl, A_dlam=A_dl, ds=ds, A_ds=self.A_rp + A_gd, dz=dz, A_dz=R["A_wt"] + self.d * A_gd + np.abs(dz))

    def dual_residual(self, dz):
        """G^T dz + c + G^T z (the dual equation of the unreduced Newton system) in high precision, per column, and
        its normwise backward-error denominator terms."""
        cols = self.Gt
        r = np.empty(self.sc_.nv)
        for j in range(self.sc_.nv):
            a, b = cols.indptr[j], cols.indptr[j + 1]
            idx, g = cols.indices[a:b], cols.data[a:b]
            r[j] = math.sumprod(list(g) + list(g) + [1.0], list(dz[idx]) + list(self.z[idx]) + [self.c[j]])
        return r


def lengths(s, z, ds, dz, eta):
    """The library's step lengths from its own ds, dz: alpha = eta / max(0, max -ds / s) if that exceeds eta, else 1
    (fmax semantics: a row at z = 0 with dz = 0 gives NaN, which is dropped)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        ms = np.fmax.reduce(np.r_[0.0, -ds / s])
        mz = np.fmax.reduce(np.r_[0.0, -dz / z])
    return (eta / ms if ms > eta else 1.0), (eta / mz if mz > eta else 1.0)


def residual_exact(M, x, b):
    """b - M x per row, each correctly rounded from exactly computed products (math.sumprod)."""
    x = list(np.asarray(x, np.float64)) + [-1.0]
    return np.array([-math.sumprod(list(M[i]) + [b[i]], x) for i in range(len(b))])


def backward_error(M, x, b):
    """Normwise backward error |b - M x|_inf / (|M|_inf |x|_inf + |b|_inf) of a solution of M x = b."""
    r = residual_exact(M, x, b)
    den = np.abs(M).sum(1).max() * np.abs(x).max() + np.abs(b).max()
    return float(np.abs(r).max() / den) if den > 0 else float(np.abs(r).max() > 0) * np.inf


def _ratio(got, want, A):
    """max |got - want| / (u A); inf where got is not finite."""
    got = np.asarray(got, np.float64)
    if not np.all(np.isfinite(got)):
        return np.inf
    err = np.abs(got - np.asarray(want, np.float64))
    return float((err / np.maximum(U * np.asarray(A, np.float64), np.finfo(float).tiny)).max()) if err.size else 0.0


def _same(a, b):
    return bool(np.array_equal(np.asarray(a), np.asarray(b)))


def check(D, sc, state, mutate=()):
    """A library step D (r3d_debug_transavg_l1_step's dict, or emulate()'s) against the float64 reference at its start
    state.  Returns (ratios: quantity -> worst |got - ref| / (u A), or the backward error over u; exact: quantity ->
    whether a bit-exact identity held)."""
    y, lam, s, z = state
    R = Step(sc, y, lam, s, z, mutate)
    N = sc.N
    q, ex = {}, {}
    nv, nA = R.norms()
    q["norms"] = max(_ratio(D["norms"][i], nv[i], nA[i]) for i in range(5))
    A = D["A"]
    low = np.tril(np.ones((N, N), bool))
    low[:N - 1, :N - 1] = True  # the T block is written in full
    q["matrix"] = _ratio(A[:N][low], R.Mred[low], R.A_Mred[low])
    ex["upper_gamma_column_zero"] = not A[:N - 1, N - 1].any()
    Rp = R.rhs(s * z, np.abs(s * z))
    q["rhs_pred"] = _ratio(A[N], Rp["red"], Rp["A_red"])
    d = np.diagonal(A[:N])
    want_sc = np.where(d > 0, 1.0 / np.sqrt(np.where(d > 0, d, 1.0)), 1.0)
    q["sc"] = _ratio(D["sc"], want_sc, want_sc)  # relative, in units of u
    Ms, bs, _ = scaled_system(A)
    k = D["retries"]
    Mf = regularised(Ms, k)
    delta = REG_REL * REG_GROWTH ** (k - 1) * np.fmax.reduce(np.r_[0.0, np.diagonal(Ms)]) if k else 0.0
    out, allow = {}, {}
    for ph, Rh in (("pred", Rp), ("corr", None)):
        P = D[ph]
        if ph == "corr":
            nr = float(sc.nr)
            mu = D["norms"][3] / nr
            rm = (D["pred"]["complementarity"] / nr) / mu
            ex["sigma"] = D["sigma"] == (rm * rm) * rm
            dsa, dza = D["pred"]["ds"], D["pred"]["dz"]
            rc = (s * z + dsa * dza) - D["sigma"] * mu
            A_rc = np.abs(s * z) + np.abs(dsa * dza) + np.abs(D["sigma"] * mu)
            Rh = R.rhs(rc, A_rc, wt_rc=(s * z) if "corrector_wt" in R.mut else None)
            q["rhs_corr"] = _ratio(P["rhs"], Rh["red"] * D["sc"], Rh["A_red"] * D["sc"] + np.abs(Rh["red"] * D["sc"]))
            b = P["rhs"]
        else:
            b = bs
        xs = P["dy"] / D["sc"]
        q["bwd_" + ph] = backward_error(Mf, xs, b) / U
        # a regularised factorisation refined once against the unregularised system leaves a residual of at most
        # 2 delta |x| (delta: what the retry added to the diagonal)
        allow["bwd_" + ph] = 2.0 * delta * np.abs(xs).max() / (np.abs(Mf).sum(1).max() * np.abs(xs).max() + np.abs(b).max()) / U
        out[ph] = (xs, b)
        Bk = R.back(P["dy"], P["dlam"], Rh)
        q["dlam_" + ph] = _ratio(P["dlam"], Bk["dlam"], Bk["A_dlam"])
        q["ds_" + ph] = _ratio(P["ds"], Bk["ds"], Bk["A_ds"])
        q["dz_" + ph] = _ratio(P["dz"], Bk["dz"], Bk["A_dz"])
        # the dual equation of the unreduced system, scaled as the reduced one (T, gamma by sc; lambda by 1 / sqrt V)
        w = np.ones(sc.nv)
        w[sc.xidx()] = D["sc"]
        w[sc.lidx()] = 1.0 / np.sqrt(R.V)
        rdual = R.dual_residual(P["dz"]) * w
        den = (np.abs(R.Gmt.multiply(w[:, None])).sum(1).max() * np.abs(P["dz"]).max() +
               np.abs(w * (R.c + R.Gt @ z)).max())
        q["dual_" + ph] = float(np.abs(rdual).max() / den / U)
        allow["dual_" + ph] = 2.0 * delta * np.abs(xs).max() / den / U
        eta = 1.0 if ph == "pred" else ETA
        ex["alpha_" + ph] = (P["alpha_p"], P["alpha_d"]) == lengths(s, z, P["ds"], P["dz"], eta)
    ap, ad = D["pred"]["alpha_p"], D["pred"]["alpha_d"]
    sa, za = s + ap * D["pred"]["ds"], z + ad * D["pred"]["dz"]
    q["complementarity"] = _ratio(D["pred"]["complementarity"], math.fsum(sa * za),
                                  math.fsum((np.abs(s) + np.abs(ap * D["pred"]["ds"])) * (np.abs(z) + np.abs(ad * D["pred"]["dz"]))))
    C = D["corr"]
    ap, ad = C["alpha_p"], C["alpha_d"]
    y1, l1, s1, z1 = D["state"]
    ex["update"] = (_same(y1, y + ap * C["dy"]) and _same(l1, lam + ap * C["dlam"]) and _same(s1, s + ap * C["ds"]) and
                    _same(z1, z + ad * C["dz"]))
    return q, ex, dict(Mf=Mf, allow=allow, solutions=out)


def bars(sc):
    """c per quantity: twice the number of additions in the longest sum the library forms for it (the host's own
    rounding is of the same order).  The one-CTA reductions (256 threads) add ceil(ne / 256) terms per thread, then 8
    tree levels; a diagonal block of the reduced system adds over the view's incident edges; the solves' normwise
    backward errors scale with N.  Worst ratios of an H100 run over the scenes of test_gpu_transavg_l1_step.py (c in
    brackets for the 300-view problem, where the largest ratios were met): norms 100 (384), matrix 168 (982), right-hand
    sides 0.49, sc 0, complementarity 2.4, dlam / ds / dz 1.9, backward errors 13 (8 N = 7184), dual equation 2.5e3
    (7184; a state with three retries, on the 60-view graph, where 8 N = 1424), exact entries 3.9 and norms 3.3."""
    red = -(-sc.ne // 256) + 8
    deg = int(np.bincount(sc.ij.ravel(), minlength=sc.m).max())
    c_sys = 2.0 * (deg + red + 8)
    return {"norms": 2.0 * (red + 8), "matrix": c_sys, "rhs_pred": c_sys, "rhs_corr": c_sys, "sc": 2.0,
            "complementarity": 2.0 * (-(-sc.nr // 256) + 8 + 4), "dlam_pred": 32.0, "dlam_corr": 32.0, "ds_pred": 32.0,
            "ds_corr": 32.0, "dz_pred": 32.0, "dz_corr": 32.0, "bwd_pred": 8.0 * sc.N, "bwd_corr": 8.0 * sc.N,
            "dual_pred": 8.0 * sc.N, "dual_corr": 8.0 * sc.N}


def over_bar(q, ex, sc, allow=None):
    """The quantities over their bars; allow: what a regularised factorisation adds to a solve's residual (check())."""
    b = bars(sc)
    allow = allow or {}
    bad = []
    for k, v in q.items():
        lim = b[k] + allow.get(k, 0.0)
        if not v <= lim:
            bad.append("%s %.3g > %.3g" % (k, v, lim))
    bad += ["%s not bit-exact" % k for k, v in ex.items() if not v]
    return bad


# ---- a stand-in for the library's step, in float64 (the CPU tests of the bars) ------------------------------------
def emulate(sc, state, tolerance=1e-9):
    """One iteration computed as the library computes it (dense scaled Cholesky, one refinement step against the
    unregularised system, up to 5 retries), returned in r3d_debug_transavg_l1_step's layout."""
    import scipy.linalg
    y, lam, s, z = (np.asarray(a, np.float64) for a in state)
    R = Step(sc, y, lam, s, z)
    N, nr = sc.N, float(sc.nr)
    nv, _ = R.norms()
    A = np.zeros((N + 1, N))
    A[:N] = np.tril(R.Mred)
    A[:N - 1, :N - 1] = R.Mred[:N - 1, :N - 1]
    Rp = R.rhs(s * z, np.abs(s * z))
    A[N] = Rp["red"]
    D = dict(m=sc.m, ne=sc.ne, N=N, norms=nv, A=A, not_pd=[False] * 6, retries=0, converged=False, failed=False)
    D["state0"] = (y, lam, s, z)
    pres, dres, dobj, gam = nv[0], nv[2], nv[4], y[-1]
    if pres <= tolerance * 2.0 and dres <= tolerance and abs(gam - dobj) <= tolerance * (1.0 + abs(gam)):
        D["converged"] = True
        return D
    Ms, bs, scv = scaled_system(A)
    D["sc"] = scv
    fac = None
    for k in range(REG_TRIES + 1):
        try:
            fac = scipy.linalg.cho_factor(regularised(Ms, k), lower=True)
            break
        except np.linalg.LinAlgError:
            D["not_pd"][k] = True
            if k < REG_TRIES:
                D["retries"] += 1
    if fac is None:
        D["failed"] = True
        return D

    def solve(b):
        xs = scipy.linalg.cho_solve(fac, b)
        return scv * (xs + scipy.linalg.cho_solve(fac, b - Ms @ xs))

    def phase(Rh, b, eta):
        dy = solve(b)
        dl = (Rh["rl"] - R.Mxl.T @ dy) / R.V
        gd = R.Gm @ sc.full(dy, dl)
        ds, dz = -R.rp - gd, Rh["wt"] + R.d * gd
        ap, ad = lengths(s, z, ds, dz, eta)
        return dict(dy=dy, dlam=dl, ds=ds, dz=dz, alpha_p=ap, alpha_d=ad)

    P = phase(Rp, bs, 1.0)
    P["complementarity"] = math.fsum((s + P["alpha_p"] * P["ds"]) * (z + P["alpha_d"] * P["dz"]))
    mu = nv[3] / nr
    rm = (P["complementarity"] / nr) / mu
    D["sigma"] = sig = (rm * rm) * rm
    Rc = R.rhs((s * z + P["ds"] * P["dz"]) - sig * mu, 0.0)
    bc = scv * Rc["red"]
    C = phase(Rc, bc, ETA)
    C["rhs"] = bc
    D["pred"], D["corr"] = P, C
    ap, ad = C["alpha_p"], C["alpha_d"]
    D["state"] = (y + ap * C["dy"], lam + ap * C["dlam"], s + ap * C["ds"], z + ad * C["dz"])
    return D


# ---- exact ---------------------------------------------------------------------------------------------------------
def _solve_exact(M, b):
    """Gaussian elimination in Fractions (M square, nonsingular)."""
    n = len(b)
    a = [[Fraction(v) for v in row] + [Fraction(bb)] for row, bb in zip(M, b)]
    for k in range(n):
        p = next(i for i in range(k, n) if a[i][k] != 0)
        a[k], a[p] = a[p], a[k]
        for i in range(k + 1, n):
            if a[i][k] != 0:
                f = a[i][k] / a[k][k]
                a[i] = [x - f * yk for x, yk in zip(a[i], a[k])]
    x = [Fraction(0)] * n
    for k in range(n - 1, -1, -1):
        x[k] = (a[k][n] - sum((a[k][j] * x[j] for j in range(k + 1, n)), Fraction(0))) / a[k][k]
    return x


def exact(sc, state, A_dev=None, retries=0):
    """Exact values at a state: the reduced matrix Mred and predictor right-hand side, the five norms, and (given the
    library's unscaled output A_dev and its retry count) the exact refined solution of the scaled system it factored:
    x1 = F b + F (b - M_s F b), F = (M_s regularised retries times)^-1, which is M_s^-1 b without retries."""
    y, lam, s, z = (np.asarray(a, np.float64) for a in state)
    F = Fraction
    x = sc.full(y, lam)
    xf = [F(v) for v in x]
    sf, zf = [F(v) for v in s], [F(v) for v in z]
    rows = sc.rows()
    xi = list(sc.xidx())
    pos = {c: i for i, c in enumerate(xi)}
    N = sc.N
    Mred = [[F(0)] * N for _ in range(N)]
    rhs = [F(0)] * N
    rhs[N - 1] = F(-1)  # -c_gamma
    pmax, viol, gtz = F(0), F(0), [F(0)] * sc.nv
    gtz[-1] = F(1)
    for e in range(sc.ne):
        local = {}
        rl = F(0)
        Mx = {}
        V = F(0)
        lamc = sc.nt + e
        rh = {}
        for r in range(7 * e, 7 * e + 7):
            row = [(j, F(v)) for j, v in rows[r]]
            gx = sum((g * xf[j] for j, g in row), F(0)) - (F(-1) if r % 7 == 6 else F(0))
            rp = gx + sf[r]
            pmax = max(pmax, abs(rp))
            viol = max(viol, gx)
            d = zf[r] / sf[r]
            v = zf[r] + (zf[r] * rp - sf[r] * zf[r]) / sf[r]
            for j, g in row:
                gtz[j] += g * zf[r]
                rh[j] = rh.get(j, F(0)) - g * v
                for k2, g2 in row:
                    if j == lamc and k2 == lamc:
                        V += g * d * g2
                    elif k2 == lamc:
                        Mx[j] = Mx.get(j, F(0)) + g * d * g2
                    elif j != lamc:
                        local[(j, k2)] = local.get((j, k2), F(0)) + g * d * g2
        rl = rh.pop(lamc)
        for (j, k2), val in local.items():
            Mred[pos[j]][pos[k2]] += val
        for j, a in Mx.items():
            for k2, b in Mx.items():
                Mred[pos[j]][pos[k2]] -= a * b / V
            rhs[pos[j]] -= a * rl / V
        for j, val in rh.items():
            rhs[pos[j]] += val
    norms = [pmax, max(viol, F(0)), max(abs(g) for g in gtz), sum((a * b for a, b in zip(sf, zf)), F(0)), sum(zf[6::7], F(0))]
    out = dict(Mred=Mred, rhs=rhs, norms=norms)
    if A_dev is not None:
        Ms, bs, _ = scaled_system(A_dev)
        Mf = regularised(Ms, retries)
        x0 = _solve_exact(Mf, bs)
        if retries:
            r = [F(bs[i]) - sum((F(Ms[i][j]) * x0[j] for j in range(N)), F(0)) for i in range(N)]
            x0 = [a + b for a, b in zip(x0, _solve_exact(Mf, r))]
        out["xs"] = x0
        out["kappa"] = float(np.linalg.cond(Mf))
    return out
