"""An independent restatement of what the AC-RANSAC scoring computes, in plain Python and numpy: the residual of each
model as an exact rational of its double inputs (fractions.Fraction), the same residual in float64, and the NFA curve
of a model with exact log10 binomials (math.lgamma).  Nothing here comes from the library; only its inputs do.

Models (the library's internal ids): 0 = F, symmetric epipolar error; 1 = H, asymmetric transfer error; 2 = E, given as
F = K2^-T E K1^-1, one-sided epipolar distance in pixels; 3 = P = K [R | t] (3 x 4), reprojection error."""
import math
from fractions import Fraction

import numpy as np

FLT_EPSILON = float(np.finfo(np.float32).eps)
MIN_SAMPLES = {0: 7, 1: 4, 2: 5, 3: 3}
MAX_MODELS = {0: 3, 1: 1, 2: 10, 3: 4}
MODEL_SIZE = {0: 9, 1: 9, 2: 9, 3: 12}
MULT_ERROR = {0: 0.5, 1: 1.0, 2: 0.5, 3: 1.0}  # point-to-line models take the square root of the area ratio


def exact_residual(model, F, a, b, z=0.0):
    """The residual of one point as a Fraction, or None where it is undefined (a zero denominator, a non-finite entry).
    F: the model's doubles, a = (x1, y1), b = (x2, y2), z: the point's third coordinate (model 3)."""
    vals = list(F) + list(a) + list(b) + [z]
    if not all(math.isfinite(v) for v in vals):
        return None
    F = [Fraction(v) for v in F]
    ax, ay = Fraction(a[0]), Fraction(a[1])
    bx, by = Fraction(b[0]), Fraction(b[1])
    if model in (1, 3):
        if model == 3:
            Z = Fraction(z)
            hx = F[0] * ax + F[1] * ay + F[2] * Z + F[3]
            hy = F[4] * ax + F[5] * ay + F[6] * Z + F[7]
            hw = F[8] * ax + F[9] * ay + F[10] * Z + F[11]
        else:
            hx = F[0] * ax + F[1] * ay + F[2]
            hy = F[3] * ax + F[4] * ay + F[5]
            hw = F[6] * ax + F[7] * ay + F[8]
        if hw == 0:
            return None
        return (bx - hx / hw) ** 2 + (by - hy / hw) ** 2
    l0 = F[0] * ax + F[1] * ay + F[2]  # the epipolar line F x1 in image 2
    l1 = F[3] * ax + F[4] * ay + F[5]
    l2 = F[6] * ax + F[7] * ay + F[8]
    y = bx * l0 + by * l1 + l2
    A = l0 * l0 + l1 * l1
    if A == 0:
        return None
    if model == 2:
        return y * y / A
    m0 = F[0] * bx + F[3] * by + F[6]  # F^T x2 in image 1
    m1 = F[1] * bx + F[4] * by + F[7]
    B = m0 * m0 + m1 * m1
    if B == 0:
        return None
    return y * y * (1 / A + 1 / B) / 4


def float_residuals(model, F, x1, x2, x3=None):
    """The same residuals of all points in float64 (a stand-in where exact rationals would be too slow)."""
    F = np.asarray(F, np.float64)
    with np.errstate(all="ignore"):
        if model in (1, 3):
            P = F.reshape(3, 4) if model == 3 else np.c_[F.reshape(3, 3)[:, :2], np.zeros(3), F.reshape(3, 3)[:, 2]]
            Xh = np.c_[x1, x3 if model == 3 else np.zeros(len(x1)), np.ones(len(x1))]
            h = Xh @ P.T
            d = x2 - h[:, :2] / h[:, 2:3]
            return (d * d).sum(1)
        Fm = F.reshape(3, 3)
        l = np.c_[x1, np.ones(len(x1))] @ Fm.T
        m = np.c_[x2, np.ones(len(x2))] @ Fm
        y = (np.c_[x2, np.ones(len(x2))] * l).sum(1)
        A = l[:, 0] ** 2 + l[:, 1] ** 2
        if model == 2:
            return y * y / A
        B = m[:, 0] ** 2 + m[:, 1] ** 2
        return y * y * (1 / A + 1 / B) / 4


def log10_binom(n, k):
    if k < 0 or k > n:
        return float("-inf")
    return (math.lgamma(n + 1) - math.lgamma(k + 1) - math.lgamma(n - k + 1)) / math.log(10.0)


def nfa_curve(model, residuals, M, max_thr, logalpha0):
    """NFA(k) for k = NS + 1 .. #{e <= max_thr} over the ascending residuals (k -> value dict):
    loge0 + (logalpha0 + m log10(e_(k) + FLT_EPSILON)) (k - NS) + log10 C(M, k) + log10 C(k, NS)."""
    ns = MIN_SAMPLES[model]
    e = np.sort(np.asarray(residuals, np.float64))
    e = e[e <= max_thr]
    loge0 = math.log10(MAX_MODELS[model] * (M - ns)) if M > ns else float("nan")
    out = {}
    for k in range(ns + 1, len(e) + 1):
        la = logalpha0 + MULT_ERROR[model] * math.log10(float(e[k - 1]) + FLT_EPSILON)
        out[k] = loge0 + la * (k - ns) + log10_binom(M, k) + log10_binom(k, ns)
    return out


def best_nfa(curve):
    """(minimum, first argmin) of an NFA curve; (+inf, None) when it is empty."""
    if not curve:
        return float("inf"), None
    k = min(curve, key=lambda j: (curve[j], j))
    return curve[k], k


def nfa_term_scale(model, residuals, M, max_thr, logalpha0):
    """The largest magnitude of the terms of any NFA(k): what a few ulp per term are relative to."""
    ns = MIN_SAMPLES[model]
    e = np.sort(np.asarray(residuals, np.float64))
    e = e[e <= max_thr]
    if len(e) <= ns:
        return 1.0
    la = abs(logalpha0) + MULT_ERROR[model] * np.abs(np.log10(e + FLT_EPSILON)).max()
    return 1.0 + la * (len(e) - ns) + 2 * abs(log10_binom(M, M // 2)) + abs(math.log10(max(MAX_MODELS[model] * (M - ns), 1)))
