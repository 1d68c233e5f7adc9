"""Reference of one step of r3d_rotation_averaging_l1 (what r3d_debug_rotavg_l1_step returns), built from the
optimisation problems themselves rather than from the library's per-row formulas.

On the kept component (m views, E edges (a < b), n = m - 1 free views): A is the 3E x 3n graph matrix, row 3e + k with
-1 at (a, k) and +1 at (b, k), local 0's columns dropped, columns component-major (k n + a - 1) as the library stores
its variables.  The residuals are b_e = log(R_b^T R_ab R_a) (scipy's Rotation), the update R_v exp([x_v]x).

L1RA's inner problem is the LP  min sum u  s.t.  f1 = A x - b - u <= 0,  f2 = -A x + b - u <= 0, which l1-magic's
l1decode_pd solves by Newton steps on the perturbed KKT function
    F_tau(x, u, l1, l2) = (r_dual, r_cent),  r_dual = (A^T (l1 - l2), 1 - l1 - l2),  r_cent = (-l1 f1 - 1/tau, -l2 f2 - 1/tau)
(the residual norm that l1-magic's line search measures takes A^T (l1 - l2) as the state carries it, Atv, updated by
steps rather than recomputed; the Newton step is that of F_tau as a function of the state).  KKT forms the Jacobian of F_tau as a sparse
(3n + 9E) matrix and solves J d = -F_tau unreduced; its Schur complement onto x is A^T diag(sigma) A with sigma the
elimination of each row's 3 x 3 (u, l1, l2) block, which KKT.sigma writes without cancellation.  The ratio test, the
backtracking line search and the next tau follow from their definitions.  IRLS: Geman-McClure weights
w = rho'(r) / (2 r) for rho(r) = r^2 / (r^2 + sigma^2), and the weighted least-squares step by scipy.sparse.linalg.

Two precisions:
  exact()     fractions.Fraction on the float64 inputs (scenes of at most about 12 views): the assembled Laplacians and
              right-hand sides, the norms, and the exact solution of each system the library factored.
  KKT, Irls   float64, every value with a magnitude A: the same sum taken over the absolute values of its terms.  A
              kernel that is right to round-off lands within a small multiple of u A; one that drops or misplaces a
              term does not.
check_pd() / check_irls() hold a library step (or emulate_pd() / emulate_irls()'s stand-in for one) to the reference and
return the worst ratio per quantity and the bit-exact decisions (the ratio test's minima, the trial steps, accept or
backtrack, the next tau and state), recomputed from the step's own direction.
"""
import math
from fractions import Fraction

import numpy as np
import scipy.linalg
import scipy.sparse as sp
import scipy.sparse.linalg
from scipy.spatial.transform import Rotation

U = np.finfo(np.float64).eps / 2
PD_MU, PD_ALPHA, PD_BETA, PD_MAX_BACKTRACKS, PD_TOL, PD_MAX_ITER = 10.0, 0.01, 0.5, 32, 1e-3, 50
MUTANTS = ("du_sig2_sign", "dl1_no_tinv", "rhs_hi_orientation", "diag_free_only", "step_099_twice", "irls_weight_power")
IRLS_MUTANTS = ("irls_weight_power",)


class Scene:
    """The kept component as the kernels see it: m views, per edge its local (a, b), a < b, and R_ab (R_b = R_ab R_a)."""

    def __init__(self, m, ab, Rk):
        self.m = int(m)
        self.ab = np.asarray(ab, np.int64).reshape(-1, 2)
        self.Rk = np.asarray(Rk, np.float64).reshape(-1, 3, 3)
        self.E = len(self.ab)
        self.n = self.m - 1
        self.nr, self.nv = 3 * self.E, 3 * self.n
        r, c, v = [], [], []
        for e, (a, b) in enumerate(self.ab):
            for k in range(3):
                for view, sgn in ((a, -1.0), (b, 1.0)):
                    if view > 0:
                        r.append(3 * e + k); c.append(k * self.n + view - 1); v.append(sgn)
        self.A = sp.csr_matrix((v, (r, c)), shape=(self.nr, self.nv))
        self.At = self.A.T.tocsr()
        self.absA, self.absAt = abs(self.A).tocsr(), abs(self.At).tocsr()
        self.deg = np.bincount(self.ab.ravel(), minlength=self.m)

    @classmethod
    def from_device(cls, D):
        return cls(D["m"], D["ab"], D["Rk"])

    def laplacian(self, w):
        """(A^T diag(w) A, its magnitude |A|^T diag(|w|) |A|) as dense (3, n, n): the product of the matrices."""
        L = (self.At @ sp.diags(w) @ self.A).toarray()
        Lm = (self.absAt @ sp.diags(np.abs(w)) @ self.absA).toarray()
        blk = lambda M: np.stack([M[k * self.n:(k + 1) * self.n, k * self.n:(k + 1) * self.n] for k in range(3)])
        return blk(L), blk(Lm)

    def per_component(self, v):
        return np.asarray(v).reshape(3, self.n)


# ---- rotations -------------------------------------------------------------------------------------------------------
def residuals(sc, R):
    """b (3E: row 3e + k) = log(R_b^T R_ab R_a) by scipy, and the magnitude of each entry: the log map's conditioning
    (theta / 2) / sin(theta / 2), at most pi / 2 away from theta = 2 pi, times the 9 terms of each product entry."""
    a, b = sc.ab[:, 0], sc.ab[:, 1]
    Em = np.einsum("eji,ejk,ekl->eil", R[b], sc.Rk, R[a])
    rv = Rotation.from_matrix(Em).as_rotvec()
    th = np.linalg.norm(rv, axis=1)
    cond = np.where(th > 1e-8, (th / 2) / np.maximum(np.sin(th / 2), 1e-300), 1.0)
    return rv.ravel(), np.repeat(9.0 * (1.0 + cond), 3)


def rotate(R, x, n):
    """R_v exp([x_v]x) (scipy), x component-major; local 0 unchanged."""
    out = np.array(R, np.float64, copy=True)
    X = np.asarray(x).reshape(3, n).T
    out[1:] = np.einsum("vij,vjk->vik", R[1:], Rotation.from_rotvec(X).as_matrix())
    return out


# ---- the L1 problem's Newton step --------------------------------------------------------------------------------------
def unpack(state):
    return tuple(np.asarray(s, np.float64) for s in state)


class KKT:
    """l1decode_pd's Newton step at a state (x, Ax, u, l1, l2, Atv) and tau, on the residuals b (the library's)."""

    def __init__(self, sc, b, state, tau):
        self.sc, self.b, self.tau = sc, np.asarray(b, np.float64), float(tau)
        self.x, self.Ax, self.u, self.l1, self.l2, self.Atv = unpack(state)
        self.tinv = 1.0 / self.tau
        # the constraints at the state, as the LP defines them (A x as the state carries it)
        self.f1 = (self.Ax - self.b) - self.u
        self.f2 = (-self.Ax + self.b) - self.u
        # sigma: the Schur complement of the row block [[0, -1, -1], [l1, -f1, 0], [l2, 0, -f2]] onto x, which is
        # 4 l1 l2 / (l1 |f2| + l2 |f1|) (every term positive inside the interior)
        l1, l2, g1, g2 = self.l1, self.l2, -self.f1, -self.f2
        self.sigma = 4.0 * l1 * l2 / (l1 * g2 + l2 * g1)
        self.A_sigma = 2.0 * (l1 / g1 + l2 / g2)  # what the device's sum and cancelling difference are bounded by

    def residual_vector(self, Atv, l1, l2, f1, f2):
        """F_tau, split in its parts: r_dual_x (3n), r_dual_u, r_cent1, r_cent2 (3E each), and their magnitudes."""
        t = self.tinv
        F = (Atv, (1.0 - l1) - l2, -l1 * f1 - t, -l2 * f2 - t)
        Am = (np.abs(Atv), 1.0 + np.abs(l1) + np.abs(l2), np.abs(l1 * f1) + t, np.abs(l2 * f2) + t)
        return F, Am

    def norms(self, Atv=None, l1=None, l2=None, f1=None, f2=None, tinv=None):
        """(sdg, |F_tau|) at a point (default: the state) and magnitudes for sdg and |F|^2."""
        Atv = self.Atv if Atv is None else Atv
        l1, l2 = (self.l1, self.l2) if l1 is None else (l1, l2)
        f1, f2 = (self.f1, self.f2) if f1 is None else (f1, f2)
        keep = self.tinv
        if tinv is not None:
            self.tinv = tinv
        F, Am = self.residual_vector(Atv, l1, l2, f1, f2)
        self.tinv = keep
        sq = math.fsum(np.concatenate([v * v for v in F]))
        A_sq = math.fsum(np.concatenate([v * v for v in Am]))
        sdg = -math.fsum(np.concatenate([f1 * l1, f2 * l2]))
        A_sdg = math.fsum(np.concatenate([np.abs(f1 * l1), np.abs(f2 * l2)]))
        return sdg, math.sqrt(sq), A_sdg, A_sq

    def jacobian(self):
        """The Jacobian of F_tau in (dx, du, dl1, dl2) order, sparse, and -F_tau with its magnitude (r_dual_x =
        A^T (l1 - l2) from the matrix)."""
        sc = self.sc
        A, At = sc.A, sc.At
        Ir = sp.identity(sc.nr, format="csr")
        Z = None
        L1, L2, F1, F2 = (sp.diags(v) for v in (self.l1, self.l2, self.f1, self.f2))
        J = sp.bmat([[Z, Z, At, -At],
                     [Z, Z, -Ir, -Ir],
                     [-L1 @ A, L1, -F1, Z],
                     [L2 @ A, L2, Z, -F2]], format="csr")
        dv = self.l1 - self.l2
        F, Am = self.residual_vector(sc.At @ dv, self.l1, self.l2, self.f1, self.f2)
        Am = (sc.absAt @ np.abs(dv),) + Am[1:]
        return J, -np.concatenate(F), np.concatenate(Am)

    def solve(self):
        """The Newton step from the unreduced system: dx, du, dl1, dl2."""
        J, rhs, _ = self.jacobian()
        d = scipy.sparse.linalg.spsolve(J.tocsc(), rhs)
        nv, nr = self.sc.nv, self.sc.nr
        return d[:nv], d[nv:nv + nr], d[nv + nr:nv + 2 * nr], d[nv + 2 * nr:]

    def reduced(self):
        """The reduced system (A^T diag(sigma) A) dx = r as (3, n, n) Laplacians and (3, n) right-hand sides, each
        with its magnitude.  r = A^T rho: the x rows of -F_tau minus the eliminated rows' share, which per row is
        rho = ((a - c) / (a + c)) w2 - (1/tau) (1/|f1| - 1/|f2|), a = l1 / |f1|, c = l2 / |f2|,
        w2 = 1/tau (1/|f1| + 1/|f2|) - 1 (the -A^T (l1 - l2) of the x rows cancels against the rows' -l1 + l2)."""
        sc, t = self.sc, self.tinv
        g1, g2 = -self.f1, -self.f2
        a, c = self.l1 / g1, self.l2 / g2
        w2 = t * (1.0 / g1 + 1.0 / g2) - 1.0
        A_w2 = t * (1.0 / g1 + 1.0 / g2) + 1.0
        rho = ((a - c) / (a + c)) * w2 - t * (1.0 / g1 - 1.0 / g2)
        A_rho = 2.0 * A_w2 + t * (1.0 / g1 + 1.0 / g2)  # the device's (sig2 / sig1) w2 carries sig1's cancellation
        r = sc.At @ rho
        A_r = sc.absAt @ A_rho
        L, Lm = sc.laplacian(self.sigma)
        Lm_sig = (sc.absAt @ sp.diags(self.A_sigma) @ sc.absA).toarray()
        Lm = np.stack([Lm_sig[k * sc.n:(k + 1) * sc.n, k * sc.n:(k + 1) * sc.n] for k in range(3)])
        return L, Lm, sc.per_component(r), sc.per_component(A_r)

    def kkt_residual(self, dx, du, dl1, dl2):
        """J d + F_tau for a direction, per block, with the magnitude of each equation: |J| |d| + |F| with |dl1|, |dl2|
        replaced by the magnitudes of what each is made of once the row is solved for it (third and fourth block
        rows: l1 (A dx - du) / |f1| + l1 + (1/tau) / |f1|, and likewise), so that a direction that cancels there is
        held to the precision its terms allow."""
        J, mF, Am = self.jacobian()
        sc, t = self.sc, self.tinv
        d = np.concatenate([dx, du, dl1, dl2])
        r = J @ d - mF
        Adx = np.abs(sc.A @ dx)
        g1, g2 = -self.f1, -self.f2
        m1 = self.l1 * (Adx + np.abs(du)) / g1 + self.l1 + t / g1
        m2 = self.l2 * (Adx + np.abs(du)) / g2 + self.l2 + t / g2
        dm = np.concatenate([np.abs(dx), np.abs(du), np.maximum(m1, np.abs(dl1)), np.maximum(m2, np.abs(dl2))])
        Jm = abs(J) @ dm + Am
        nv = sc.nv
        return r[:nv], Jm[:nv], r[nv:], Jm[nv:]

    def trial(self, dx, Adx, du, dl1, dl2, Atdv, s):
        """The trial point at step s (the update as the LP's variables move) and its F_tau norm."""
        xp, Axp, up = self.x + s * dx, self.Ax + s * Adx, self.u + s * du
        l1p, l2p, Atvp = self.l1 + s * dl1, self.l2 + s * dl2, self.Atv + s * Atdv
        f1, f2 = (Axp - self.b) - up, (-Axp + self.b) - up
        return (xp, Axp, up, l1p, l2p, Atvp), self.norms(Atvp, l1p, l2p, f1, f2)


def ratio_test(f1, f2, l1, l2, Adx, du, dl1, dl2):
    """Per edge min(1, the largest step keeping l1, l2 > 0 and f1, f2 < 0 along (d f1, d f2) = (A dx - du, -A dx - du)),
    from the definition, in IEEE double on the given direction."""
    g1, g2 = Adx - du, -Adx - du
    with np.errstate(divide="ignore", invalid="ignore"):
        cands = [np.where(dl1 < 0, -l1 / dl1, np.inf), np.where(dl2 < 0, -l2 / dl2, np.inf),
                 np.where(g1 > 0, -f1 / g1, np.inf), np.where(g2 > 0, -f2 / g2, np.inf)]
    r = np.minimum(1.0, np.min(np.stack(cands), axis=0))
    return r.reshape(-1, 3).min(axis=1)


def _ratio(got, want, A):
    got = np.asarray(got, np.float64)
    if not np.all(np.isfinite(got)):
        return np.inf
    err = np.abs(got - np.asarray(want, np.float64))
    return float((err / np.maximum(U * np.asarray(A, np.float64), np.finfo(float).tiny)).max()) if err.size else 0.0


def _two_prod(a, b):
    """a b = p + e exactly (Dekker's product with Veltkamp's split; no FMA needed)."""
    p = a * b
    c = 134217729.0 * a
    ah = c - (c - a)
    al = a - ah
    c = 134217729.0 * b
    bh = c - (c - b)
    bl = b - bh
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    return p, e


def backward_error(L, x, r):
    """Normwise backward error |r - L x|_inf / (|L|_inf |x|_inf + |r|_inf), each residual correctly rounded from the
    exact products."""
    L, x, r = (np.asarray(v, np.float64) for v in (L, x, r))
    p, e = _two_prod(L, x[None, :])
    rr = np.array([math.fsum(np.r_[r[i], -p[i], -e[i]]) for i in range(len(r))])
    den = np.abs(L).sum(1).max() * np.abs(x).max() + np.abs(r).max()
    return float(np.abs(rr).max() / den) if den > 0 else 0.0


def bars(sc):
    """c per quantity: twice the number of additions in the longest sum the library forms for it.  The 1024-thread
    reductions add ceil(P / 1024) terms per thread (P = max(E, n)), then 10 tree levels, each term itself a sum of
    up to 9; a Laplacian entry sums over the view's incident edges; the solves' normwise backward errors scale with n.
    Worst ratios of an H100 run over the scenes of test_gpu_rotavg_l1_step.py: b 1.8, sigx 2.9, laplacian 9.5 (bench300,
    c = 606), rhs 0, sdg 4.8, resnorm and trial_resnorm 3.9, kkt_rows 2.0, kkt_x 5.8, bwd 2.9, rotation 1.3, w 0."""
    red = -(-max(sc.E, sc.n) // 1024) + 10 + 9
    deg = int(sc.deg.max())
    return {"b": 16.0, "sdg": 2.0 * red, "resnorm": 2.0 * red, "sigx": 16.0, "laplacian": 2.0 * (deg + 4),
            "rhs": 2.0 * (deg + 8), "bwd": 8.0 * max(sc.n, 1), "kkt_x": 16.0 * max(sc.n, 1), "kkt_rows": 64.0,
            "Atdv": 2.0 * (deg + 2), "trial_resnorm": 2.0 * red, "rotation": 16.0, "w": 8.0, "wb": 8.0}


# ---- checks ----------------------------------------------------------------------------------------------------------
def _laplacian_checks(D, L, Lm, r, A_r, q, key="laplacian", rkey="rhs"):
    """The device's (3, n + 1, n) assembled systems against the reference Laplacians and right-hand sides."""
    lap = np.asarray(D["laplacians"])
    n = L.shape[1]
    q[key] = max(_ratio(lap[k, :n], L[k], Lm[k]) for k in range(3))
    q[rkey] = max(_ratio(lap[k, n], r[k], A_r[k]) for k in range(3))
    q["bwd"] = max(backward_error(lap[k, :n], np.asarray(D["dx"]).reshape(3, n)[k], lap[k, n]) / U for k in range(3))


def check_pd(D, sc, b, state, tau):
    """A kind-0 step D (r3d_debug_rotavg_l1_step's dict or emulate_pd()'s) against the reference at its start state.
    Returns (ratios: quantity -> worst |got - ref| / (u A), or a backward error over u; exact: decision -> held)."""
    K = KKT(sc, b, state, tau)
    q, ex = {}, {}
    sdg, res, A_sdg, A_sq = K.norms()
    if "sdg0" in D:
        q["sdg"] = _ratio(D["sdg0"], sdg, A_sdg)
        q["resnorm"] = _ratio(D["resnorm0"] ** 2, res * res, A_sq)
    if "sigx" in D:
        q["sigx"] = _ratio(D["sigx"], K.sigma, K.A_sigma)
    L, Lm, r, A_r = K.reduced()
    # inside the interior every sigma > 0, so on a connected graph each Laplacian is positive definite
    ex["positive_definite"] = not D["not_pd"]
    if D["not_pd"]:
        if "laplacians" in D:
            lap = np.asarray(D["laplacians"])
            q["laplacian"] = max(_ratio(lap[k, :sc.n], L[k], Lm[k]) for k in range(3))
        return q, ex
    dx = np.asarray(D["dx"], np.float64)
    if "laplacians" in D:
        _laplacian_checks(D, L, Lm, r, A_r, q)
    Adx, du, dl1, dl2, Atdv = (np.asarray(D[k], np.float64) for k in ("Adx", "du", "dl1", "dl2", "Atdv"))
    ex["Adx"] = bool(np.array_equal(Adx, sc.A @ dx))
    q["Atdv"] = _ratio(Atdv, sc.At @ (dl1 - dl2), sc.absAt @ np.abs(dl1 - dl2))
    # the direction against the unreduced Newton system: the x rows normwise, each row's (u, l1, l2) block by its own
    # largest magnitude
    rx, mx, rr, mr = K.kkt_residual(dx, du, dl1, dl2)
    q["kkt_x"] = float(np.abs(rx).max() / max(mx.max(), 1e-300) / U)
    nr = sc.nr
    blk = np.maximum(np.maximum(mr[:nr], mr[nr:2 * nr]), mr[2 * nr:])
    q["kkt_rows"] = float(max((np.abs(rr[i * nr:(i + 1) * nr]) / np.maximum(blk, 1e-300)).max() for i in range(3)) / U)
    # decisions from the device's own direction, bit for bit
    rmin = ratio_test(K.f1, K.f2, K.l1, K.l2, Adx, du, dl1, dl2)
    ex["rmin"] = bool(np.array_equal(D["rmin"], rmin))
    ex["step_max"] = D["step_max"] == min(1.0, float(rmin.min()))
    trials = D["trials"]
    s = 0.99 * D["step_max"]
    ok = True
    worst = 0.0
    for t, (st, rn) in enumerate(trials):
        ok &= st == s
        pt, (_, rref, _, asq) = K.trial(dx, Adx, du, dl1, dl2, Atdv, st)
        worst = max(worst, _ratio(rn * rn, rref * rref, asq))
        acc = rn <= (1.0 - PD_ALPHA * st) * D["resnorm0"]
        ok &= acc == (t == len(trials) - 1 and D["accepted"])
        s = PD_BETA * s
    ex["trials"] = bool(ok) and 1 <= len(trials) <= PD_MAX_BACKTRACKS + 1 and (D["accepted"] or len(trials) == PD_MAX_BACKTRACKS + 1)
    q["trial_resnorm"] = worst
    if D["accepted"] and "state" in D:
        pt, (sdg1, res1, A_sdg1, _) = K.trial(dx, Adx, du, dl1, dl2, Atdv, trials[-1][0])
        ex["state"] = all(np.array_equal(a, c) for a, c in zip(D["state"], pt))
        q["sdg_new"] = _ratio(D["sdg"], sdg1, A_sdg1)
        ex["tau"] = D["tau"] == PD_MU * (2.0 * sc.nr) / D["sdg"]
        K1 = KKT(sc, b, pt, D["tau"])
        _, res2, _, A_sq2 = K1.norms()
        q["resnorm_new"] = _ratio(D["resnorm"] ** 2, res2 * res2, A_sq2)
    return q, ex


def check_rotations(D, sc, R0, x):
    """The update R_v exp([x_v]x) against scipy, in units of u (3 terms per entry of magnitude 1), and max |x|."""
    Rn = rotate(R0, x, sc.n)
    return {"rotation": _ratio(D["rotations"], Rn, np.ones_like(Rn) * 3.0)}, {"xmax": D["xmax"] == float(np.abs(x).max(initial=0.0))}


class Irls:
    """One IRLS step at the library's residuals b: weights from the Geman-McClure loss, the weighted least-squares
    direction by scipy.sparse.linalg."""

    def __init__(self, sc, b, sigma_deg):
        self.sc, self.b = sc, np.asarray(b, np.float64)
        s2 = (sigma_deg * (math.pi / 180.0)) ** 2
        self.s2 = s2
        # rho(r) = r^2 / (r^2 + s2); rho'(r) = 2 r s2 / (r^2 + s2)^2; w = rho'(r) / (2 r)
        t = self.b * self.b + s2
        self.w = s2 / (t * t)
        self.wb = self.w * self.b

    def solve(self):
        sc = self.sc
        H = (sc.At @ sp.diags(self.w) @ sc.A).tocsc()
        return scipy.sparse.linalg.spsolve(H, sc.At @ self.wb)


def check_irls(D, sc, sigma_deg):
    """A kind-1 step D at its own residuals D["b"] against Irls: weights, assembled systems, the solves' backward
    error."""
    I = Irls(sc, D["b"], sigma_deg)
    q, ex = {}, {}
    q["w"] = _ratio(D["w"], I.w, 3.0 * I.w)
    q["wb"] = _ratio(D["wb"], I.wb, 4.0 * np.abs(I.wb))
    L, Lm = sc.laplacian(I.w)
    r = sc.per_component(sc.At @ I.wb)
    A_r = sc.per_component(sc.absAt @ (4.0 * np.abs(I.wb)))
    Lm = 3.0 * Lm
    if "laplacians" in D:
        _laplacian_checks(D, L, Lm, r, A_r, q)
    return q, ex


def over_bar(q, ex, sc):
    b = bars(sc)
    bad = ["%s %.3g > %.3g" % (k, v, b[k.replace("_new", "")]) for k, v in q.items() if not v <= b[k.replace("_new", "")]]
    return bad + ["%s not bit-exact" % k for k, v in ex.items() if not v]


# ---- a stand-in for the library's step in float64 (the CPU tests of the bars) --------------------------------------
def assemble(sc, w, v, mutate=()):
    """The systems as k_l1_system assembles them: per free view its row of each Laplacian (off-diagonal -w over edges to
    free views, diagonal the sum over all incident edges) and (A^T v) in row n."""
    n = sc.n
    lap = np.zeros((3, n + 1, n))
    W, V = np.asarray(w).reshape(-1, 3), np.asarray(v).reshape(-1, 3)
    for e, (a, b) in enumerate(sc.ab):
        for view, other in ((a, b), (b, a)):
            if view == 0:
                continue
            if other > 0:
                lap[:, view - 1, other - 1] = -W[e]
            if other > 0 or "diag_free_only" not in mutate:
                lap[:, view - 1, view - 1] += W[e]
            hi = (view == b) != ("rhs_hi_orientation" in mutate)
            lap[:, n, view - 1] += V[e] if hi else -V[e]
    return lap


def _cholesky_solve(lap):
    n = lap.shape[2]
    out = []
    for k in range(3):
        L = np.linalg.cholesky(lap[k, :n])
        y = scipy.linalg.solve_triangular(L, lap[k, n], lower=True)
        out.append(scipy.linalg.solve_triangular(L.T, y, lower=False))
    return np.concatenate(out)


def emulate_pd(sc, b, state, tau, mutate=()):
    """One Newton iteration computed the way the library's kernels compute it (per-row formulas, per-view assembly,
    dense Cholesky), in r3d_debug_rotavg_l1_step's layout.  mutate: names from MUTANTS, plausible kernel slips."""
    import scipy.linalg  # noqa: F401
    x, Ax, u, l1, l2, Atv = unpack(state)
    b = np.asarray(b, np.float64)
    tinv = 1.0 / tau
    f1, f2 = (Ax - b) - u, (-Ax + b) - u

    def norm(Atv, l1, l2, f1, f2, t):
        rd = (1.0 - l1) - l2
        rc1, rc2 = -l1 * f1 - t, -l2 * f2 - t
        return math.sqrt(math.fsum(np.r_[Atv * Atv, rd * rd + rc1 * rc1 + rc2 * rc2])), -math.fsum(np.r_[f1 * l1, f2 * l2])

    res0, sdg0 = norm(Atv, l1, l2, f1, f2, tinv)
    w2 = -1.0 - tinv * (1.0 / f1 + 1.0 / f2)
    sig1 = -l1 / f1 - l2 / f2
    sig2 = l1 / f1 - l2 / f2
    sigx = sig1 - sig2 * sig2 / sig1
    rrow = -tinv * (-1.0 / f1 + 1.0 / f2) - (sig2 / sig1) * w2
    lap = assemble(sc, sigx, rrow, mutate)
    D = dict(sdg0=sdg0, tau0=tau, resnorm0=res0, sigx=sigx, rrow=rrow, w2=w2, laplacians=lap.copy(), not_pd=False)
    try:
        dx = _cholesky_solve(lap)
    except np.linalg.LinAlgError:
        D["not_pd"] = True
        return D
    Adx = sc.A @ dx
    du = (w2 - (-sig2 if "du_sig2_sign" in mutate else sig2) * Adx) / sig1
    dl1 = -(l1 / f1) * (Adx - du) - l1 - (0.0 if "dl1_no_tinv" in mutate else tinv / f1)
    dl2 = (l2 / f2) * (Adx + du) - l2 - tinv / f2
    Atdv = sc.At @ (dl1 - dl2)
    rmin = ratio_test(f1, f2, l1, l2, Adx, du, dl1, dl2)
    step_max = float(rmin.min())
    s = 0.99 * step_max
    if "step_099_twice" in mutate:
        s = 0.99 * s
    trials, accepted = [], False
    for _ in range(PD_MAX_BACKTRACKS + 1):
        xp, Axp, up, l1p, l2p, Atvp = x + s * dx, Ax + s * Adx, u + s * du, l1 + s * dl1, l2 + s * dl2, Atv + s * Atdv
        rn, sdg = norm(Atvp, l1p, l2p, (Axp - b) - up, (-Axp + b) - up, tinv)
        trials.append((s, rn))
        if rn <= (1.0 - PD_ALPHA * s) * res0:
            accepted = True
            break
        s = PD_BETA * s
    D.update(dx=dx, Adx=Adx, du=du, dl1=dl1, dl2=dl2, Atdv=Atdv, rmin=rmin, step_max=step_max, trials=trials, accepted=accepted)
    if accepted:
        st = (xp, Axp, up, l1p, l2p, Atvp)
        tau1 = PD_MU * (2.0 * sc.nr) / sdg
        D.update(state=st, sdg=sdg, tau=tau1, resnorm=norm(Atvp, l1p, l2p, (Axp - b) - up, (-Axp + b) - up, 1.0 / tau1)[0])
    return D


def emulate_irls(sc, b, sigma_deg, mutate=()):
    s2 = (sigma_deg * (math.pi / 180.0)) ** 2
    t = b * b + s2
    w = s2 / t if "irls_weight_power" in mutate else s2 / (t * t)
    lap = assemble(sc, w, w * b)
    return dict(b=b, w=w, wb=w * b, laplacians=lap.copy(), dx=_cholesky_solve(lap))


def start_state(sc, b):
    """k_l1_pd_start's point at the residuals b (x = 0, A x = 0, u = 0.95 |b| + 0.1 max |b|, lambda = -1 / f) and its
    tau = mu 2M / sdg."""
    bm = float(np.abs(b).max())
    u = 0.95 * np.abs(b) + 0.10 * bm
    f1, f2 = (0.0 - b) - u, (-0.0 + b) - u
    l1, l2 = -1.0 / f1, -1.0 / f2
    Atv = sc.At @ (l1 - l2)
    return (np.zeros(sc.nv), np.zeros(sc.nr), u, l1, l2, Atv)


# ---- exact -----------------------------------------------------------------------------------------------------------
def _solve_exact(M, r):
    n = len(r)
    a = [[Fraction(float(v)) for v in row] + [Fraction(float(rr))] for row, rr in zip(M, r)]
    for k in range(n):
        p = next(i for i in range(k, n) if a[i][k] != 0)
        a[k], a[p] = a[p], a[k]
        for i in range(k + 1, n):
            if a[i][k] != 0:
                f = a[i][k] / a[k][k]
                a[i] = [xx - f * yk for xx, yk in zip(a[i], a[k])]
    x = [Fraction(0)] * n
    for k in range(n - 1, -1, -1):
        x[k] = (a[k][n] - sum((a[k][j] * x[j] for j in range(k + 1, n)), Fraction(0))) / a[k][k]
    return x


def exact(sc, b, state, tau, lap_dev=None):
    """Exact values at a state (Fractions of the float64 inputs, the constraint values f included): sigma per row, the
    Laplacians and right-hand sides
    (3, n + 1, n) by the Schur complement of each row's block, sdg and |F_tau|^2, and, given the library's assembled
    systems, the exact solution of each (3, n)."""
    F = Fraction
    x, Ax, u, l1, l2, Atv = unpack(state)
    b = np.asarray(b, np.float64)
    f1v, f2v = (Ax - b) - u, (-Ax + b) - u  # the constraints formed once in float64, as KKT and the library form them
    tinv = F(1) / F(float(tau))
    n = sc.n
    lap = [[[F(0)] * n for _ in range(n + 1)] for _ in range(3)]
    sq, sdg = F(0), F(0)
    atv_l = [F(0)] * sc.nv
    for e, (a, bb) in enumerate(sc.ab):
        for k in range(3):
            i = 3 * e + k
            L1, L2 = F(float(l1[i])), F(float(l2[i]))
            f1, f2 = F(float(f1v[i])), F(float(f2v[i]))
            g1, g2 = -f1, -f2
            sig = 4 * L1 * L2 / (L1 * g2 + L2 * g1)
            ca, cc = L1 / g1, L2 / g2
            w2 = tinv * (1 / g1 + 1 / g2) - 1
            rho = ((ca - cc) / (ca + cc)) * w2 - tinv * (1 / g1 - 1 / g2)
            sq += (1 - L1 - L2) ** 2 + (-L1 * f1 - tinv) ** 2 + (-L2 * f2 - tinv) ** 2
            sdg -= f1 * L1 + f2 * L2
            for view, other, sg in ((a, bb, -1), (bb, a, 1)):
                if view == 0:
                    continue
                lap[k][view - 1][view - 1] += sig
                if other > 0:
                    lap[k][view - 1][other - 1] -= sig
                lap[k][n][view - 1] += sg * rho
    for j in range(sc.nv):
        at = F(float(Atv[j]))
        sq += at * at
    out = dict(lap=lap, sq=sq, sdg=sdg)
    if lap_dev is not None:
        out["x"] = [_solve_exact(lap_dev[k, :n], lap_dev[k, n]) for k in range(3)]
    return out
