"""Float64 reference of one bundle-adjustment LM step (what r3d_debug_ba_step returns), built independently of the
library: residuals and Jacobians from the oracle's forward-mode autodiff (pyoracle.ba_jacobian_model, ba_prior), Ceres'
Huber corrector (rho'' <= 0: residual and Jacobian rows scaled by sqrt(rho')), Jacobi scaling 1 / (1 + |column|), the
LM diagonal D^2 = clamp(diag, 1e-6, 1e32) / radius, and the point Schur complement formed with sparse matrices and
vectorised 3x3 blocks (no dense H, so 200-camera problems stay cheap).

Besides the values, every quantity comes with a magnitude A: the same sum taken over absolute values of its terms.  In
it a Jacobian entry counts as |J_ij| + max_k |J_ik| and a residual as |r| + |measurement| + f, the sizes their rounding
errors scale with: the library's analytic model and the oracle's autodiff agree to about 26 ulp of a row's largest
entry and 240 ulp of a measured coordinate, not to ulps of each entry.  Each point's V^-1 counts normwise, times the
condition number of V.  A kernel that is right to round-off lands within a small multiple of u A; one that drops or
doubles a term does not."""
import numpy as np
import scipy.sparse as sp

U = np.finfo(np.float64).eps / 2


def huber_rho1(s, a):
    """rho'(s) of Ceres' HuberLoss(a) (s = squared residual norm): 1 inside, a / sqrt(s) outside."""
    s = np.asarray(s, np.float64)
    if a <= 0:
        return np.ones_like(s)
    out = s > a * a
    return np.where(out, a / np.sqrt(np.where(out, s, 1.0)), 1.0)


def jacobian(oracle, p, huber_a, refine, prior_huber_a):
    """Corrected (unscaled) Jacobian J (sparse CSR), residual r, and their magnitudes Jm, rm; plus the layout."""
    nc, ni, npt = len(p["poses"]), len(p["intrinsics"]), len(p["points"])
    nB = 6 * nc + (6 * ni if refine else 0)
    nparam = nB + 3 * npt
    model = p.get("intr_model")
    ext = p.get("intrinsics_ext")
    rows, cols, vals, mags, rs, rms = [], [], [], [], [], []
    row = 0
    for o in range(len(p["obs_xy"])):
        c, ip = int(p["obs_cam"][o]), int(p["obs_pt"][o])
        g = int(p["cam_intr"][c])
        m = 3 if model is None else int(model[g])
        r, J = oracle.ba_jacobian_model(m, p["intrinsics"][g], None if ext is None else ext[g], p["poses"][c],
                                        p["points"][ip], p["obs_xy"][o])
        sq = np.sqrt(huber_rho1(r @ r, huber_a))
        cidx = list(range(6 * c, 6 * c + 6)) + list(range(nB + 3 * ip, nB + 3 * ip + 3))
        Jk = np.concatenate([J[:, 6:12], J[:, 12:15]], 1)
        if refine:
            cidx = list(range(6 * nc + 6 * g, 6 * nc + 6 * g + 6)) + cidx
            Jk = np.concatenate([J[:, :6], Jk], 1)
        for a in range(2):
            rows += [row] * len(cidx)
            cols += cidx
            vals.append(sq * Jk[a])
            mags.append(sq * (np.abs(Jk[a]) + np.abs(J[a]).max()))
            rs.append(sq * r[a])
            rms.append(sq * (abs(r[a]) + np.abs(p["obs_xy"][o]).max() + abs(p["intrinsics"][g][0])))
            row += 1
    npri = 0 if p.get("prior_cam") is None else len(p["prior_cam"])
    for k in range(npri):
        c = int(p["prior_cam"][k])
        r, J = oracle.ba_prior(p["poses"][c], p["prior_center"][k], p["prior_weight"][k])
        sq = np.sqrt(huber_rho1(r @ r, prior_huber_a))
        cen = np.abs(p["prior_weight"][k]) * (np.abs(p["prior_center"][k]) + np.abs(p["poses"][c][3:]).sum())
        for a in range(3):
            rows += [row] * 6
            cols += list(range(6 * c, 6 * c + 6))
            vals.append(sq * J[a])
            mags.append(sq * (np.abs(J[a]) + np.abs(J[a]).max()))
            rs.append(sq * r[a])
            rms.append(sq * (abs(r[a]) + cen.max()))
            row += 1
    vals = np.concatenate(vals) if vals else np.zeros(0)
    mags = np.concatenate(mags) if mags else np.zeros(0)
    J = sp.csr_matrix((vals, (rows, cols)), shape=(row, nparam))
    Jm = sp.csr_matrix((mags, (rows, cols)), shape=(row, nparam))
    return J, np.array(rs), Jm, np.array(rms), nB, nparam, npt


def step(oracle, p, radius, huber_a=16.0, refine=1, prior_huber_a=0.0):
    """The reference step.  Returns a dict with the values r3d_debug_ba_step returns (g, diag, scale, S, rhs, Vinv,
    gmax), the magnitudes A_g, A_diag, A_S, A_rhs, A_Vinv, and what the delta checks need (H as a sparse matrix,
    D2, kappa of every V)."""
    J, r, Jm, rm, nB, nparam, npt = jacobian(oracle, p, huber_a, refine, prior_huber_a)
    du = np.asarray(J.multiply(J).sum(0)).ravel()
    gu = J.T @ r
    scale = 1.0 / (1.0 + np.sqrt(du))
    g = gu * scale
    diag = du * scale * scale
    A_g = (Jm.T @ rm) * scale
    A_diag = np.asarray(Jm.multiply(Jm).sum(0)).ravel() * scale * scale
    D2 = np.clip(diag, 1e-6, 1e32) / radius
    Sc = sp.diags(scale)
    Js, Jsm = (J @ Sc).tocsc(), (Jm @ Sc).tocsc()
    JB, JP, JmB, JmP = Js[:, :nB], Js[:, nB:], Jsm[:, :nB], Jsm[:, nB:]
    # per point: V = sum Jp^T Jp + D^2 (3x3 blocks of JP^T JP), its inverse and condition number
    HPP = (JP.T @ JP).tocoo()
    V = np.zeros((npt, 3, 3))
    np.add.at(V, (HPP.row // 3, HPP.row % 3, HPP.col % 3), HPP.data)
    V[:, [0, 1, 2], [0, 1, 2]] += D2[nB:].reshape(npt, 3)
    Vinv = np.linalg.inv(V) if npt else np.zeros((0, 3, 3))
    kappa = np.linalg.cond(V) if npt else np.zeros(0)
    # V^-1 moves by about |V^-1| |dV| |V^-1| for an error dV in V's terms, and inverting adds kappa(V) |V^-1| normwise
    HmPP = (JmP.T @ JmP).tocoo()
    Vm = np.zeros((npt, 3, 3))
    np.add.at(Vm, (HmPP.row // 3, HmPP.row % 3, HmPP.col % 3), HmPP.data)
    Vm[:, [0, 1, 2], [0, 1, 2]] += D2[nB:].reshape(npt, 3)
    A_Vinv = np.abs(Vinv) @ Vm @ np.abs(Vinv) + (kappa * np.abs(Vinv).max((1, 2)))[:, None, None]

    def blockdiag(B):
        i = np.repeat(np.arange(3 * npt), 3)
        j = (np.arange(npt)[:, None, None] * 3 + np.arange(3)[None, None, :]).repeat(3, 1).ravel()
        return sp.csr_matrix((B.ravel(), (i, j)), shape=(3 * npt, 3 * npt))

    Vi_bd, Va_bd = blockdiag(Vinv), blockdiag(A_Vinv)
    HBP, HmBP = (JB.T @ JP).tocsr(), (JmB.T @ JmP).tocsr()
    S = (JB.T @ JB).toarray() - (HBP @ Vi_bd @ HBP.T).toarray()
    S[np.arange(nB), np.arange(nB)] += D2[:nB]
    A_S = (JmB.T @ JmB).toarray() + (HmBP @ Va_bd @ HmBP.T).toarray()
    A_S[np.arange(nB), np.arange(nB)] += D2[:nB]
    rhs = -g[:nB] + HBP @ (Vi_bd @ g[nB:])
    A_rhs = A_g[:nB] + HmBP @ (Va_bd @ A_g[nB:])
    H = (Js.T @ Js).tocsr() + sp.diags(D2)
    return dict(g=g, diag=diag, scale=scale, gmax=np.abs(gu).max() if len(gu) else 0.0, S=S, rhs=rhs, Vinv=Vinv,
                A_g=A_g, A_diag=A_diag, A_S=A_S, A_rhs=A_rhs, A_Vinv=A_Vinv, H=H, D2=D2, kappa=kappa, nB=nB,
                nparam=nparam, J=J, r=r)


def cost(oracle, p, huber_a=16.0, prior_huber_a=0.0):
    """0.5 * sum rho(|r|^2) over observations and priors (the LM cost), from the oracle's residuals."""
    def rho(s, a):
        return s if a <= 0 or s <= a * a else 2 * a * np.sqrt(s) - a * a
    model, ext = p.get("intr_model"), p.get("intrinsics_ext")
    c = 0.0
    for o in range(len(p["obs_xy"])):
        cam, ip = int(p["obs_cam"][o]), int(p["obs_pt"][o])
        gi = int(p["cam_intr"][cam])
        r, _ = oracle.ba_jacobian_model(3 if model is None else int(model[gi]), p["intrinsics"][gi],
                                        None if ext is None else ext[gi], p["poses"][cam], p["points"][ip], p["obs_xy"][o])
        c += 0.5 * rho(r @ r, huber_a)
    for k in range(0 if p.get("prior_cam") is None else len(p["prior_cam"])):
        r, _ = oracle.ba_prior(p["poses"][int(p["prior_cam"][k])], p["prior_center"][k], p["prior_weight"][k])
        c += 0.5 * rho(r @ r, prior_huber_a)
    return c


def solve_reduced(ref):
    """The step from the reference's own reduced system: S dB = rhs, dP = V^-1 (-g_P - H_PB dB)."""
    nB = ref["nB"]
    dB = np.linalg.solve(ref["S"], ref["rhs"])
    H = ref["H"]
    t = -ref["g"][nB:] - H[nB:, :nB] @ dB
    dP = np.einsum("pij,pj->pi", ref["Vinv"], t.reshape(-1, 3)).ravel()
    return np.concatenate([dB, dP])
