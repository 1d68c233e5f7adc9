"""CPU restatement of r3d_rotation_averaging_l1 in float64 (numpy / scipy), for the tests and the bench.

Chatterjee & Govindu's robust rotation averaging as OpenMVG's GlobalRotationsRobust runs it, on the kept component of
the L2 method (triplet rejection, largest bi-edge-connected component; taken from orc_rotation_averaging, which selects
it by the same rules).  On kept local ids (local 0 = the lowest kept view id, held at R = I), with R_b = R_ab R_a:
  1. start: a breadth-first spanning tree from local 0, neighbours in ascending order; R_b = R_ab R_a along it.
  2. L1RA: per outer iteration, b_e = log(R_b^T R_ab R_a) (the Ceres quaternion log), x = argmin |A x - b|_1 by
     l1-magic's l1decode_pd (Candes & Romberg) from x = 0, R_v <- R_v exp([x_v]x); stop when max |x| <= tolerance.
     A: row 3e + k holds -1 at (a, k) and +1 at (b, k), local 0's columns dropped.
  3. IRLS: per iteration the residuals b, weights w = sigma^2 / (b^2 + sigma^2)^2 per row, (A^T W A) x = A^T W b,
     R_v <- R_v exp([x_v]x), the same stopping rule.
Every row of A touches one component k, so A^T diag(d) A is three weighted graph Laplacians of size m - 1, one per
component; every solve here is three Cholesky factorisations.  The arithmetic is numpy's, so this agrees with the
device to rounding, not bit for bit.
"""
import numpy as np
import scipy.linalg

from oracle import pyoracle_rotavg as rpo

PD_TOL = 1e-3           # l1decode_pd: stop when the surrogate duality gap < PD_TOL
PD_MAX_ITER = 50
PD_MU = 10.0
PD_ALPHA = 0.01         # sufficient decrease of the residual norm
PD_BETA = 0.5           # backtracking factor
PD_MAX_BACKTRACKS = 32

DEFAULTS = dict(max_angular_error_deg=5.0, irls_sigma_deg=5.0, l1_max_iterations=32, irls_max_iterations=32,
                tolerance=1e-5)


class FactorizationError(RuntimeError):
    pass


# ---- Ceres' angle-axis conversions (row-major), as the device writes them ------------------------------------------
def aa_to_R(aa):
    th2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2]
    if th2 > 2.220446049250313e-16:
        th = np.sqrt(th2)
        wx, wy, wz = aa[0] / th, aa[1] / th, aa[2] / th
        c, s = np.cos(th), np.sin(th)
        oc = 1.0 - c
        return np.array([[c + wx * wx * oc, wx * wy * oc - wz * s, wy * s + wx * wz * oc],
                         [wz * s + wx * wy * oc, c + wy * wy * oc, wy * wz * oc - wx * s],
                         [wx * wz * oc - wy * s, wx * s + wy * wz * oc, c + wz * wz * oc]])
    return np.array([[1.0, -aa[2], aa[1]], [aa[2], 1.0, -aa[0]], [-aa[1], aa[0], 1.0]])


def R_to_aa(R):
    R = np.asarray(R).ravel()
    q = np.zeros(4)
    tr = R[0] + R[4] + R[8]
    if tr >= 0.0:
        t = np.sqrt(tr + 1.0)
        q[0] = 0.5 * t
        t = 0.5 / t
        q[1], q[2], q[3] = (R[7] - R[5]) * t, (R[2] - R[6]) * t, (R[3] - R[1]) * t
    else:
        i = 0
        if R[4] > R[0]:
            i = 1
        if R[8] > R[4 * i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = np.sqrt(R[4 * i] - R[4 * j] - R[4 * k] + 1.0)
        q[i + 1] = 0.5 * t
        t = 0.5 / t
        q[0] = (R[3 * k + j] - R[3 * j + k]) * t
        q[j + 1] = (R[3 * j + i] + R[3 * i + j]) * t
        q[k + 1] = (R[3 * k + i] + R[3 * i + k]) * t
    s2 = q[1] * q[1] + q[2] * q[2] + q[3] * q[3]
    if s2 > 0.0:
        st = np.sqrt(s2)
        two_theta = 2.0 * (np.arctan2(-st, -q[0]) if q[0] < 0.0 else np.arctan2(st, q[0]))
        return q[1:] * (two_theta / st)
    return 2.0 * q[1:]


# ---- the graph matrix A (3E x 3(m - 1)), its transpose and the three Laplacians ------------------------------------
def apply_A(ab, x):
    """A x for x (m, 3) (row 0 = the held view, zero): (E, 3)."""
    return x[ab[:, 1]] - x[ab[:, 0]]


def apply_At(ab, v, m):
    """A^T v for v (E, 3): (m, 3), row 0 zero."""
    out = np.zeros((m, 3))
    np.add.at(out, ab[:, 1], v)
    np.add.at(out, ab[:, 0], -v)
    out[0] = 0.0
    return out


def solve_laplacians(ab, w, rhs, m):
    """(A^T diag(w) A) x = rhs (m, 3; row 0 ignored): per component k the Laplacian of the edge weights w[:, k] without
    row and column 0, factored by Cholesky.  Raises FactorizationError when one is not positive definite."""
    x = np.zeros((m, 3))
    a, b = ab[:, 0], ab[:, 1]
    for k in range(3):
        L = np.zeros((m, m))
        np.add.at(L, (a, a), w[:, k])
        np.add.at(L, (b, b), w[:, k])
        np.add.at(L, (a, b), -w[:, k])
        np.add.at(L, (b, a), -w[:, k])
        try:
            fac = scipy.linalg.cho_factor(L[1:, 1:], lower=True)
        except np.linalg.LinAlgError:
            raise FactorizationError()
        x[1:, k] = scipy.linalg.cho_solve(fac, rhs[1:, k])
    return x


# ---- l1decode_pd on the graph matrix ---------------------------------------------------------------------------------
def l1_regression(ab, b, m, pdtol=PD_TOL, pdmaxiter=PD_MAX_ITER, trace=None):
    """x = argmin |A x - b|_1 (x (m, 3), row 0 = 0) by l1-magic's primal-dual method on min sum u s.t. -u <= A x - b <= u,
    from x = 0, u = 0.95 |b| + 0.1 max |b|.  Returns (x, stats): iterations, backtracks (rejected trial steps), sdg
    (the final surrogate duality gap), stuck (a Newton step found no sufficient decrease in PD_MAX_BACKTRACKS halvings:
    the last iterate is returned).  b all zero: x = 0 without iterations.  Raises FactorizationError.  trace: called
    once per Newton iteration with a dict of the state it started from (x, u, Ax, Atv, lam1, lam2, tau), its direction
    (dx, du, Adx, dlam1, dlam2, Atdv), the trial steps and whether the last was accepted (the tests take states and
    steps from it)."""
    ab = np.asarray(ab, np.int64)
    b = np.asarray(b, np.float64).reshape(-1, 3)
    M = b.size
    x = np.zeros((m, 3))
    st = {"iterations": 0, "backtracks": 0, "sdg": 0.0, "stuck": False}
    bmax = np.abs(b).max() if M else 0.0
    if bmax == 0.0:
        return x, st
    Ax = np.zeros_like(b)
    u = 0.95 * np.abs(b) + 0.10 * bmax
    fu1 = (Ax - b) - u
    fu2 = (-Ax + b) - u
    lam1 = -1.0 / fu1
    lam2 = -1.0 / fu2
    Atv = apply_At(ab, lam1 - lam2, m)

    def norms(Atv, lam1, lam2, fu1, fu2, tinv):
        rd = (1.0 - lam1) - lam2
        rc1 = -lam1 * fu1 - tinv
        rc2 = -lam2 * fu2 - tinv
        return np.sqrt((Atv[1:] ** 2).sum() + (rd * rd + rc1 * rc1 + rc2 * rc2).sum())

    sdg = -((fu1 * lam1).sum() + (fu2 * lam2).sum())
    tau = PD_MU * 2.0 * M / sdg
    resnorm = norms(Atv, lam1, lam2, fu1, fu2, 1.0 / tau)
    it = 0
    while not (sdg < pdtol or it >= pdmaxiter):
        it += 1
        tinv = 1.0 / tau
        w2 = -1.0 - tinv * (1.0 / fu1 + 1.0 / fu2)
        sig1 = -lam1 / fu1 - lam2 / fu2
        sig2 = lam1 / fu1 - lam2 / fu2
        sigx = sig1 - sig2 * sig2 / sig1
        rrow = -tinv * (-1.0 / fu1 + 1.0 / fu2) - (sig2 / sig1) * w2
        dx = solve_laplacians(ab, sigx, apply_At(ab, rrow, m), m)
        Adx = apply_A(ab, dx)
        du = (w2 - sig2 * Adx) / sig1
        dlam1 = -(lam1 / fu1) * (Adx - du) - lam1 - tinv / fu1
        dlam2 = (lam2 / fu2) * (Adx + du) - lam2 - tinv / fu2
        Atdv = apply_At(ab, dlam1 - dlam2, m)
        # the largest step keeping lam > 0 and fu < 0, capped at 1
        s = 1.0
        for num, den in ((lam1, dlam1), (lam2, dlam2)):
            neg = den < 0
            if neg.any():
                s = min(s, (-num[neg] / den[neg]).min())
        for f, d in ((fu1, Adx - du), (fu2, -Adx - du)):
            pos = d > 0
            if pos.any():
                s = min(s, (-f[pos] / d[pos]).min())
        s = 0.99 * s
        steps = []
        for _ in range(PD_MAX_BACKTRACKS + 1):
            steps.append(s)
            xp = x + s * dx
            up = u + s * du
            Axp = Ax + s * Adx
            Atvp = Atv + s * Atdv
            lam1p = lam1 + s * dlam1
            lam2p = lam2 + s * dlam2
            fu1p = (Axp - b) - up
            fu2p = (-Axp + b) - up
            if norms(Atvp, lam1p, lam2p, fu1p, fu2p, tinv) <= (1.0 - PD_ALPHA * s) * resnorm:
                break
            st["backtracks"] += 1
            s = PD_BETA * s
        else:
            st["stuck"] = True
        if trace is not None:
            trace(dict(x=x, u=u, Ax=Ax, Atv=Atv, lam1=lam1, lam2=lam2, tau=tau, dx=dx, du=du, Adx=Adx, dlam1=dlam1,
                       dlam2=dlam2, Atdv=Atdv, steps=steps, accepted=not st["stuck"]))
        if st["stuck"]:
            break
        x, u, Ax, Atv, lam1, lam2, fu1, fu2 = xp, up, Axp, Atvp, lam1p, lam2p, fu1p, fu2p
        sdg = -((fu1 * lam1).sum() + (fu2 * lam2).sum())
        tau = PD_MU * 2.0 * M / sdg
        resnorm = norms(Atv, lam1, lam2, fu1, fu2, 1.0 / tau)
    st["iterations"] = it
    st["sdg"] = float(sdg)
    return x, st


# ---- the method ------------------------------------------------------------------------------------------------------
def spanning_tree_start(ab, Rab, m):
    """R (m, 3, 3): breadth-first tree from local 0 (R = I), neighbours in ascending order."""
    nbr = [[] for _ in range(m)]
    for e, (a, b) in enumerate(ab):
        nbr[a].append((b, e))
        nbr[b].append((a, e))
    R = np.zeros((m, 3, 3))
    R[0] = np.eye(3)
    seen = np.zeros(m, bool)
    seen[0] = True
    queue = [0]
    for v in queue:
        for w, e in sorted(nbr[v]):
            if seen[w]:
                continue
            seen[w] = True
            R[w] = Rab[e] @ R[v] if ab[e][0] == v else Rab[e].T @ R[v]
            queue.append(w)
    return R


def residuals(ab, Rab, R):
    """b (E, 3): log(R_b^T R_ab R_a)."""
    return np.array([R_to_aa(R[b].T @ (Rab[e] @ R[a])) for e, (a, b) in enumerate(ab)]).reshape(-1, 3)


def rotate(R, x):
    return np.array([R[v] @ aa_to_R(x[v]) for v in range(len(R))])


def kept_problem(rel, n_views, max_angular_error_deg=5.0):
    """The L2 method's kept component (orc_rotation_averaging, no refinement): (view_kept, edge_kept, edge_support,
    summary, ab (E, 2) local ids a < b in (a, b) order, Rab (E, 3, 3) with R_b = R_ab R_a, kept view ids)."""
    _, vk, ek, sup, S = rpo.rotation_averaging(rel, n_views, refine=False, max_angular_error_deg=max_angular_error_deg)
    views = np.nonzero(vk)[0]
    local = np.full(n_views, -1)
    local[views] = np.arange(len(views))
    recs = np.nonzero(ek)[0]
    I, J = local[rel["I"][recs].astype(int)], local[rel["J"][recs].astype(int)]
    Rr = np.asarray(rel["rotation"][recs], np.float64).reshape(-1, 3, 3)
    a, b = np.minimum(I, J), np.maximum(I, J)
    Rab = np.where((I < J)[:, None, None], Rr, Rr.transpose(0, 2, 1))
    order = np.lexsort((b, a))
    return vk, ek, sup, S, np.stack([a, b], 1)[order], Rab[order], views


def solve(ab, Rab, m, irls_sigma_deg=5.0, l1_max_iterations=32, irls_max_iterations=32, tolerance=1e-5, start=None):
    """Steps 1-3 on kept local ids: (R (m, 3, 3), summary dict).  start: rotations to begin from in place of the
    spanning tree's (the tests use it to start away from the truth)."""
    ab = np.asarray(ab, np.int64)
    R = spanning_tree_start(ab, Rab, m) if start is None else np.array(start, np.float64)
    S = {"l1_iterations": 0, "pd_iterations": 0, "pd_backtracks": 0, "irls_iterations": 0, "termination": 1}
    S["initial_l1_cost"] = float(np.abs(residuals(ab, Rab, R)).sum())
    try:
        for _ in range(l1_max_iterations):
            x, st = l1_regression(ab, residuals(ab, Rab, R), m)
            S["pd_iterations"] += st["iterations"]
            S["pd_backtracks"] += st["backtracks"]
            R = rotate(R, x)
            S["l1_iterations"] += 1
            if np.abs(x).max() <= tolerance:
                S["termination"] = 0
                break
        if irls_max_iterations > 0:
            S["termination"] = 1
            s2 = np.radians(irls_sigma_deg) ** 2
            for _ in range(irls_max_iterations):
                b = residuals(ab, Rab, R)
                t = b * b + s2
                w = s2 / (t * t)
                x = solve_laplacians(ab, w, apply_At(ab, w * b, m), m)
                R = rotate(R, x)
                S["irls_iterations"] += 1
                if np.abs(x).max() <= tolerance:
                    S["termination"] = 0
                    break
    except FactorizationError:
        S["termination"] = 2
    S["final_l1_cost"] = float(np.abs(residuals(ab, Rab, R)).sum())
    return R, S


def rotation_averaging_l1(rel, n_views, max_angular_error_deg=5.0, irls_sigma_deg=5.0, l1_max_iterations=32,
                          irls_max_iterations=32, tolerance=1e-5):
    """The library's call restated: (rotations (n_views, 3, 3), view_kept, edge_kept, edge_support, summary dict).
    Raises ValueError for invalid options and pyoracle_rotavg.OracleError for invalid records."""
    if not (l1_max_iterations >= 1 and irls_max_iterations >= 0 and tolerance > 0.0 and irls_sigma_deg > 0.0):
        raise ValueError("invalid options")
    vk, ek, sup, S0, ab, Rab, views = kept_problem(rel, n_views, max_angular_error_deg)
    rot = np.zeros((n_views, 3, 3))
    summ = {k: S0[k] for k in ("success", "n_edges", "n_triplets", "n_valid_triplets", "n_kept_edges", "n_kept_views")}
    summ.update(l1_iterations=0, pd_iterations=0, pd_backtracks=0, irls_iterations=0, termination=-1,
                initial_l1_cost=0.0, final_l1_cost=0.0)
    if not S0["success"]:
        return rot, vk, ek, sup, summ
    R, S = solve(ab, Rab, len(views), irls_sigma_deg, l1_max_iterations, irls_max_iterations, tolerance)
    summ.update(S)
    rot[views] = R
    return rot, vk, ek, sup, summ
