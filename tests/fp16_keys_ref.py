"""Float64 reference of the fp16 candidate path: k_view_prepare's operands, the distance surrogate they encode, the
real distances, their chunk minima and the error bound eps_pair the certification relies on (DESIGN.md 2.1); and
check_pair, which holds a device's operands and candidate keys to them term by term.

The bound is restated from DESIGN.md here, not read back from the library, so a change to the library's pair_eps
cannot move the reference with it."""
import numpy as np

CHUNK = 8          # database rows per candidate key (r3d::kChunk)
BIAS_COLS = 16     # the K-step holding the norm terms (r3d::kBiasCols)
ROW_PAD = 256      # views are padded to a multiple of this many rows (r3d::kRowPad)
COL_ALIGN = 64     # operand rows are padded to a multiple of this many halves
PAD_P0 = 65504.0   # p0 of a padding row of the database role: it loses against every real row


def pad_up(x, m):
    return (x + m - 1) // m * m


def n_pad(n):
    return pad_up(max(n, 1), ROW_PAD)


def kmain(dim):
    return pad_up(dim, 16)


def operand_cols(dim):
    return pad_up(kmain(dim) + BIAS_COLS, COL_ALIGN)


def k16_steps(dim):
    """k16 MMA steps of one distance: the descriptor's, then the one holding the norms."""
    return (kmain(dim) + BIAS_COLS) // 16


def chunk_bits(nI):
    """Low mantissa bits of a key that hold the chunk id (match_host.cu: at least 4)."""
    nchunks, bits = n_pad(nI) // CHUNK, 4
    while (1 << bits) < nchunks:
        bits += 1
    return bits


def kernel_norm2(desc, kcols):
    """||a||^2 of every row in float64, summed in k_view_prepare's order: lane l adds a_k^2 for k = l, l + 32, ...
    (k < kcols, zero beyond the descriptor), then the xor butterfly over 16, 8, 4, 2, 1 lanes."""
    a = np.zeros((len(desc), pad_up(kcols, 32)), np.float64)
    a[:, :desc.shape[1]] = desc.astype(np.float32)
    sq = (a * a).reshape(len(desc), -1, 32)
    lane = sq[:, 0, :].copy()
    for r in range(1, sq.shape[1]):
        lane = lane + sq[:, r, :]
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        lane = lane + lane[:, idx ^ o]
    return lane[:, 0]


def norm_split(n2, e0):
    """(p0, p1) as fp16 with ||a||^2 ~= p0 * 2^e0 + p1 * 2^(e0 - 11); both divisions and roundings as the kernel does
    them (double -> half, round to nearest even)."""
    S0, S1 = np.ldexp(1.0, e0), np.ldexp(1.0, e0 - 11)
    p0 = (n2 / S0).astype(np.float16)
    r = n2 - p0.astype(np.float64) * S0
    p1 = (r / S1).astype(np.float16)
    return p0, p1


def split_value(p0, p1, e0):
    return p0.astype(np.float64) * np.ldexp(1.0, e0) + p1.astype(np.float64) * np.ldexp(1.0, e0 - 11)


def prepare(desc, e0):
    """k_view_prepare restated: (opQ, opD), n_pad x kp float16 (compare bit patterns: signed zeros matter).
    opD row = [fp16(a) 0.. | p0 p1 S0 S1 0..], opQ row = [fp16(-2 fp16(a)) -0.. | S0 S1 p0 p1 0..] (the columns up to
    kmain = pad16(dim)); padding rows: opQ zero, opD = [0.. | 65504 0 S0 S1 0..]."""
    n, dim = desc.shape
    km, kp, npd = kmain(dim), operand_cols(dim), n_pad(n)
    S0, S1 = np.float16(np.ldexp(1.0, e0)), np.float16(np.ldexp(1.0, e0 - 11))
    opQ = np.zeros((npd, kp), np.float16)
    opD = np.zeros((npd, kp), np.float16)
    h = np.zeros((n, km), np.float16)
    h[:, :dim] = desc.astype(np.float32).astype(np.float16)
    opD[:n, :km] = h
    opQ[:n, :km] = (np.float32(-2.0) * h.astype(np.float32)).astype(np.float16)  # -0 for the zero columns, as on the device
    p0, p1 = norm_split(kernel_norm2(desc, km), e0)
    opD[:n, km], opD[:n, km + 1], opD[:n, km + 2], opD[:n, km + 3] = p0, p1, S0, S1
    opQ[:n, km], opQ[:n, km + 1], opQ[:n, km + 2], opQ[:n, km + 3] = S0, S1, p0, p1
    opD[n:, km], opD[n:, km + 2], opD[n:, km + 3] = np.float16(PAD_P0), S0, S1
    return opQ, opD


def view_stats(desc):
    """The four quantities k_view_stats reduces, in float64: max ||a||^2, max ||fp16(a)||^2, max ||a - fp16(a)||^2,
    max |a_k| (zeros for an empty view)."""
    if len(desc) == 0:
        return np.zeros(4)
    a = desc.astype(np.float32).astype(np.float64)
    h = desc.astype(np.float32).astype(np.float16).astype(np.float64)
    return np.array([(a * a).sum(1).max(), (h * h).sum(1).max(), ((a - h) ** 2).sum(1).max(), np.abs(a).max()])


def eps_terms(stats_db, stats_q, e0, dim):
    """The three terms of eps_pair (DESIGN.md 2.1) for database view I and query view J of dimension dim, from
    view_stats: quantisation 2 (max||a - fp16(a)|| max||b|| + max||fp16(a)|| max||b - fp16(b)||),
    split 2^-21 (max||a||^2 + max||b||^2) + 2^(e0-35) (two rows, each within 2^-22 ||a||^2 + 2^(e0-36)),
    accumulation 2^-21 max(8, k16 steps) (max||a|| + max||b||)^2."""
    nI, hI, dI = np.sqrt(stats_db[:3])
    nJ, _, dJ = np.sqrt(stats_q[:3])
    quant = 2.0 * (dI * nJ + hI * dJ)
    split = np.ldexp(nI * nI + nJ * nJ, -21) + np.ldexp(1.0, e0 - 35)
    acc = np.ldexp(max(8, k16_steps(dim)) * (nI + nJ) ** 2, -21)
    return quant, split, acc


def eps_pair(stats_db, stats_q, e0, dim):
    return float(sum(eps_terms(stats_db, stats_q, e0, dim)))


def surrogate(opQ_q, opD_db):
    """The value the tensor cores approximate, exactly: opQ(J) . opD(I)^T, nJ x nI_pad (fp16 products are exact in
    float64, the sums round far below any bound of interest)."""
    return opQ_q.astype(np.float64) @ opD_db.astype(np.float64).T


def real_distances(db, q):
    """||b - a||^2 in float64, nJ x nI."""
    A = db.astype(np.float32).astype(np.float64)
    B = q.astype(np.float32).astype(np.float64)
    return np.maximum((B * B).sum(1)[:, None] + (A * A).sum(1)[None, :] - 2.0 * B @ A.T, 0.0)


def chunk_minima(D, nI):
    """Minimum over every CHUNK consecutive database columns of D (columns >= nI do not exist: +inf)."""
    nq, cols = D.shape
    full = np.full((nq, n_pad(nI)), np.inf)
    full[:, :min(cols, nI)] = D[:, :nI]
    return full.reshape(nq, -1, CHUNK).min(2)


def unpack_keys(keys, bits):
    """Candidate keys (uint32) -> (float value with the chunk bits, float value with them cleared, chunk id)."""
    keys = np.ascontiguousarray(keys, np.uint32)
    mask = np.uint32((1 << bits) - 1)
    kv = keys.view(np.float32).astype(np.float64)
    masked = (keys & ~mask).view(np.float32).astype(np.float64)
    return kv, masked, (keys & mask).astype(np.int64)


def check_pair(ctx, I, J, db, q, label):
    """The fp16 candidate bound of (database view I, query view J) on the device, term by term, against this reference;
    returns the largest measured share of each term.
    1. The operands equal prepare() bit for bit; the device's stats are upper bounds of view_stats().
    2. Every row's norm split is within 2^-21 max||a||^2 + 2^(e0-36); the quantisation error of every pair is within its
       term.
    3. Every key, chunk bits cleared, is within the accumulation term + 2^(b-23)|key| of the surrogate minimum of the
       chunk its low bits name; the library's eps_pair is at least eps_pair() here.
    4. Certification (k = 2, stage A; k = 5, stage B): every chunk outside keys 0..k-1 has a real minimum
       >= kv_k - 2^(b-23)|kv_k| - eps_pair."""
    nI, nJ, dim = len(db), len(q), db.shape[1]
    oI, oJ = ctx.debug_view_operands(I), ctx.debug_view_operands(J)
    e0 = oI["e0"]
    assert oJ["e0"] == e0
    assert oI["opD"] is not None and oJ["opQ"] is not None, "%s: the views should take the fp16 path" % label
    km = kmain(dim)
    out = {}
    # 1. operands bit for bit, stats as upper bounds of the float64 values
    stats = []
    for v, o in ((db, oI), (q, oJ)):
        rQ, rD = prepare(v, e0)
        assert np.array_equal(o["opQ"].view(np.uint16), rQ.view(np.uint16)), "%s: opQ differs" % label
        assert np.array_equal(o["opD"].view(np.uint16), rD.view(np.uint16)), "%s: opD differs" % label
        s, st = view_stats(v), o["stats"].astype(np.float64)
        assert (st[:3] >= s[:3] * (1 - 2.0 ** -40)).all() and st[3] == s[3], (label, st, s)
        assert s[0] < 2.0 ** (e0 + 13)        # p0 <= 2^13: the split's first piece stays in fp16 range
        stats.append(s)
    sI, sJ = stats
    quant, split, acc = eps_terms(sI, sJ, e0, dim)
    eps = quant + split + acc
    # 2. norm split of every row (the device's p0, p1) against the budget the pair term gives one row
    worst, worst_rel = 0.0, 0.0
    for v, o, s in ((db, oI, sI), (q, oJ, sJ)):
        n2 = (v.astype(np.float64) ** 2).sum(1)
        err = np.abs(split_value(o["opD"][:len(v), km], o["opD"][:len(v), km + 1], e0) - n2)
        budget = np.ldexp(s[0], -21) + np.ldexp(1.0, e0 - 36)
        assert (err <= budget).all(), "%s: split error %g over %g" % (label, err.max(), budget)
        worst = max(worst, err.max() / budget)
        worst_rel = max(worst_rel, err.max() / max(np.ldexp(s[0], -21), 1e-300))
    out["split"], out["split_without_floor"] = worst, worst_rel
    # quantisation: |a.b - fp16(a).fp16(b)| over all pairs against its term
    A, B = db.astype(np.float32).astype(np.float64), q.astype(np.float32).astype(np.float64)
    hA, hB = [x.astype(np.float32).astype(np.float16).astype(np.float64) for x in (db, q)]
    qerr = 2.0 * np.abs(B @ A.T - hB @ hA.T).max()
    assert qerr <= quant + 2.0 ** -40 * (np.sqrt(sI[0] * sJ[0]) + 1e-300), (label, qerr, quant)
    out["quant"] = qerr / quant if quant > 0 else float("nan")
    # 3. accumulation: every key against the float64 surrogate minimum of the chunk its low bits name
    keys, eps_lib = ctx.debug_candidate_keys(I, J, nJ)
    assert eps_lib >= eps * (1 - 1e-6), "%s: the library's eps_pair %g is below the bound's %g" % (label, eps_lib, eps)
    bits = chunk_bits(nI)
    kv, masked, cid = unpack_keys(keys[:nJ, :6], bits)
    assert (np.diff(kv, axis=1) >= 0).all() and (np.sort(cid, 1)[:, 1:] != np.sort(cid, 1)[:, :-1]).all()
    S = surrogate(oJ["opQ"][:nJ], oI["opD"]).reshape(nJ, -1, CHUNK).min(2)
    s_at = np.take_along_axis(S, cid, 1)
    trunc = np.ldexp(np.abs(kv), bits - 23)             # clearing the chunk bits moves the value by less than this
    dev = np.abs(masked - s_at)
    assert (dev <= acc + trunc).all(), "%s: key off its surrogate by %g (slack %g)" % (label, (dev - trunc).max(), acc)
    # the accumulator's own error, between these two bounds, over the chunks that hold real rows
    real = cid * CHUNK < nI
    out["acc_lo"] = max(0.0, (dev - trunc)[real].max()) / acc if acc > 0 else 0.0
    out["acc_hi"] = (dev + trunc)[real].max() / acc if acc > 0 else float("nan")
    # 4. the certification invariant, stage A (k = 2) and stage B (k = 5)
    Rc = chunk_minima(real_distances(db, q), nI)
    rows = np.arange(nJ)[:, None]
    share = -np.inf
    for k in (2, 5):
        other = Rc.copy()
        other[rows, cid[:, :k]] = np.inf
        m = other.min(1)
        lb = kv[:, k] - np.ldexp(np.abs(kv[:, k]), bits - 23) - eps
        assert (m >= lb).all(), "%s: a chunk outside keys 0..%d is closer than LB(key %d)" % (label, k - 1, k)
        fin = np.isfinite(m)
        if fin.any():
            share = max(share, ((kv[:, k] - np.ldexp(np.abs(kv[:, k]), bits - 23) - m)[fin]).max() / eps)
    out["cert"] = share
    print("%-34s e0=%3d eps=%.3e quant=%.3f split=%.3f (no floor %.3g) acc=[%.3f, %.3f] cert=%.3f" % (
        label, e0, eps, out["quant"], out["split"], out["split_without_floor"], out["acc_lo"], out["acc_hi"], out["cert"]))
    return out
