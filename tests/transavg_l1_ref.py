"""CPU restatement of r3d_translation_averaging_l1 in float64 (numpy / scipy.sparse), for the tests and the bench.

The linear program of Moulon et al. (ICCV 2013) on the kept edges: variables y = (T of the free kept views, lambda per
edge, gamma), minimise gamma subject to -gamma <= (T_J - R_IJ T_I - lambda u_IJ)_k <= gamma and lambda >= 1, the lowest
kept view held at T = 0.  Written as min c^T y s.t. G y + s = h, s >= 0 (7 rows per edge) and solved by the same
Mehrotra predictor-corrector as the library: the same start, step rule, centring and stopping test, the same
elimination of each lambda, the same Jacobi scaling of the (T, gamma) system before its dense Cholesky and the same
step of iterative refinement of every solve against the unregularised system.  Its arithmetic is numpy's (sparse
products, LAPACK Cholesky), so it agrees with the device to rounding, not bit for bit.

The kept edges and views are those of orc_translation_averaging (oracle/oracle_transavg.cpp), which selects them by the
same rules.
"""
import numpy as np
import scipy.linalg
import scipy.sparse as sp

from oracle import pyoracle_transavg as pto

ETA = 0.99
REG_REL = 1e-18
REG_GROWTH = 100.0
REG_TRIES = 5


def kept_edges(rel, rotations, rot_kept, n_views, edge_use=None):
    """(view_kept, edge_kept) of orc_translation_averaging (one LM iteration: only its selection is used)."""
    _, _, vk, ek, S = pto.translation_averaging(rel, rotations, rot_kept, n_views, edge_use=edge_use, max_iterations=1)
    return vk, ek, S


def build_lp(rel, rotations, view_kept, edge_kept):
    """The LP of the kept edges: (G (csr), h, c, kept view ids, kept record ids).  Columns: 3 per free kept view in view
    id order, one lambda per kept record in record order, gamma last."""
    views = np.nonzero(view_kept)[0]
    recs = np.nonzero(edge_kept)[0]
    local = np.full(len(view_kept), -1)
    local[views] = np.arange(len(views))
    m, ne = len(views), len(recs)
    nt = 3 * (m - 1)
    nv = nt + ne + 1
    R = np.asarray(rotations, np.float64).reshape(-1, 3, 3)
    I = local[rel["I"][recs].astype(int)]
    J = local[rel["J"][recs].astype(int)]
    Rij = np.einsum("eab,ecb->eac", R[rel["J"][recs].astype(int)], R[rel["I"][recs].astype(int)])
    t = rel["translation"][recs]
    u = t / np.linalg.norm(t, axis=1, keepdims=True)
    rows, cols, vals = [], [], []
    for e in range(ne):
        for k in range(3):
            # r_k = T_J[k] - R[k, :] T_I - lambda u_k; rows 6e + k: r_k - gamma, 6e + 3 + k: -r_k - gamma
            terms = []
            if J[e] > 0:
                terms.append((3 * (J[e] - 1) + k, 1.0))
            if I[e] > 0:
                terms += [(3 * (I[e] - 1) + c, -Rij[e, k, c]) for c in range(3)]
            terms.append((nt + e, -u[e, k]))
            for sign, row in ((1.0, 7 * e + k), (-1.0, 7 * e + 3 + k)):
                for col, v in terms:
                    rows.append(row); cols.append(col); vals.append(sign * v)
                rows.append(row); cols.append(nv - 1); vals.append(-1.0)
        rows.append(7 * e + 6); cols.append(nt + e); vals.append(-1.0)
    G = sp.csr_matrix((vals, (rows, cols)), shape=(7 * ne, nv))
    h = np.zeros(7 * ne)
    h[6::7] = -1.0
    c = np.zeros(nv)
    c[-1] = 1.0
    return G, h, c, views, recs


def solve(G, h, c, n_free, max_iterations=100, tolerance=1e-9, trace=None):
    """Mehrotra predictor-corrector on min c^T y s.t. G y + s = h, s >= 0; the first n_free coordinates of y are the
    views' translations, then one lambda per edge (7 rows each), then gamma.  Returns (y, summary dict).  trace: called
    as trace(iteration, y, s, z) with the state each iteration starts from (the tests take late states from it)."""
    nr, nv = G.shape
    ne = nr // 7
    x_idx = np.r_[np.arange(n_free), nv - 1]          # the dense system: T and gamma
    l_idx = np.arange(n_free, n_free + ne)            # eliminated: lambda
    y = np.zeros(nv)
    y[l_idx] = 2.0
    y[-1] = 3.0
    s = h - G @ y
    z = np.ones(nr)
    Gt = G.T.tocsr()
    hn = np.abs(h).max()
    term, nreg, it = 1, 0, 0
    while True:
        if trace is not None:
            trace(it, y.copy(), s.copy(), z.copy())
        rp = G @ y + s - h
        rd = c + Gt @ z
        gam, dobj = y[-1], -h @ z
        pres, dres = np.abs(rp).max(), np.abs(rd).max()
        if pres <= tolerance * (1.0 + hn) and dres <= tolerance and abs(gam - dobj) <= tolerance * (1.0 + abs(gam)):
            term = 0
            break
        if it == max_iterations:
            break
        d = z / s
        M = (Gt @ sp.diags(d) @ G).tocsc()
        Mxx = M[x_idx][:, x_idx].toarray()
        Mxl = M[x_idx][:, l_idx].tocsr()
        V = M[l_idx][:, l_idx].diagonal()
        Mred = Mxx - (Mxl @ sp.diags(1.0 / V) @ Mxl.T).toarray()
        dg = Mred.diagonal()
        sc = np.where(dg > 0, 1.0 / np.sqrt(np.where(dg > 0, dg, 1.0)), 1.0)
        Ms = Mred * sc[:, None] * sc[None, :]   # scaled to a unit diagonal
        fac = None
        for k in range(REG_TRIES + 1):
            try:
                A = Ms if k == 0 else Ms + REG_REL * REG_GROWTH ** (k - 1) * Ms.diagonal().max() * np.eye(len(x_idx))
                fac = scipy.linalg.cho_factor(A, lower=True)
                break
            except np.linalg.LinAlgError:
                if k < REG_TRIES:
                    nreg += 1
        if fac is None:
            term = 2
            break

        def step(rc):
            wt = (z * rp - rc) / s
            rhs = -(c + Gt @ (z + wt))
            rl = rhs[l_idx]
            b = sc * (rhs[x_idx] - Mxl @ (rl / V))
            xs = scipy.linalg.cho_solve(fac, b)
            xs = xs + scipy.linalg.cho_solve(fac, b - Ms @ xs)   # one refinement step against the unregularised system
            dx = sc * xs
            dy = np.zeros(nv)
            dy[x_idx] = dx
            dy[l_idx] = (rl - Mxl.T @ dx) / V
            gd = G @ dy
            return dy, -rp - gd, wt + d * gd

        def lengths(ds, dz, eta):
            ms = max(0.0, (-ds / s).max())
            mz = max(0.0, (-dz / z).max())
            return (eta / ms if ms > eta else 1.0), (eta / mz if mz > eta else 1.0)

        mu = s @ z / nr
        _, ds_a, dz_a = step(s * z)
        ap, ad = lengths(ds_a, dz_a, 1.0)
        sigma = (((s + ap * ds_a) @ (z + ad * dz_a)) / nr / mu) ** 3
        dy, ds, dz = step(s * z + ds_a * dz_a - sigma * mu)
        ap, ad = lengths(ds, dz, ETA)
        y = y + ap * dy
        s = s + ap * ds
        z = z + ad * dz
        it += 1
    viol = max(0.0, (G @ y - h).max())
    return y, {"iterations": it, "termination": term, "regularized_factorizations": nreg, "gamma": float(y[-1]),
               "dual_objective": float(-h @ z), "max_primal_violation": float(viol), "max_dual_violation": float(dres)}


def translation_averaging_l1(rel, rotations, rot_kept, n_views, edge_use=None, max_iterations=100, tolerance=1e-9):
    """The library's call restated: (centers, translations, view_kept, edge_kept, edge_scale, summary dict).  Raises
    ValueError for max_iterations < 1 or tolerance not > 0, and pyoracle_transavg.OracleError for invalid records."""
    if not max_iterations >= 1 or not tolerance > 0.0:
        raise ValueError("max_iterations < 1 or tolerance not > 0")
    vk, ek, S0 = kept_edges(rel, rotations, rot_kept, n_views, edge_use)
    cen = np.zeros((n_views, 3))
    tra = np.zeros((n_views, 3))
    lam = np.zeros(len(rel))
    summ = {"success": S0["success"], "n_edges": S0["n_edges"], "n_kept_edges": S0["n_kept_edges"],
            "n_kept_views": S0["n_kept_views"], "iterations": 0, "termination": -1, "regularized_factorizations": 0,
            "gamma": 0.0}
    if not S0["success"]:
        return cen, tra, vk, ek, lam, summ
    G, h, c, views, recs = build_lp(rel, rotations, vk, ek)
    nf = 3 * (len(views) - 1)
    y, S = solve(G, h, c, nf, max_iterations, tolerance)
    summ.update(S)
    R = np.asarray(rotations, np.float64).reshape(-1, 3, 3)
    T = np.vstack([np.zeros(3), y[:nf].reshape(-1, 3)])
    tra[views] = T
    cen[views] = -np.einsum("vba,vb->va", R[views], T)
    lam[recs] = y[nf:nf + len(recs)]
    return cen, tra, vk, ek, lam, summ
