"""CPU replay of the uint8 candidate kernel's key insertion (k_l2_candidates.cu, integer path) on seeded C3 items.

    python scripts/replay_u8_insertion.py [--pairs 4] [--items 3]

It reproduces the consumer's lane/chunk mapping: warp w of an item holds query rows 16 w .. 16 w + 15, set 0 rows
16 w + 0..7 and set 1 rows 16 w + 8..15, four lanes per row, and in half h of tile t lane q tests the chunks
t * 32 + h * 16 + 4 g + q (g = 0..3) against an integer bound on its bracket minima (bracket_bound_not).  A round
loop runs until no lane of the warp has a passed chunk left, and in round i each lane inserts its i-th chunk in the
kernel's order (passed chunks first, highest g first), so lanes with fewer passed chunks insert failed ones; a set
keeps its 6 smallest keys.  Per rule it reports the chunks that pass per warp-half,
the insertion-network executions per warp-half and the histogram of insertion rounds, and it checks that the keys
the quad merges at the end of the item are the exact top 6 of the row.

Rules:
  lane         each lane's bound is its own set's largest key; one round loop for both sets (every round runs both
               networks)
  quad         U = min(min_l key_l[5], max_l key_l[1]) over the quad, taken per half; one round loop for both sets
  quad+split   the quad bound per half; one round loop per set
  quad/tile    the quad bound taken once per tile (in the first half); one round loop per set
  union6       the exact 6th-smallest key of the quad's union, per half; one round loop per set
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

CHUNK = 8
NUM_KEYS = 6
TILE = 256
ITEM_ROWS = 256
PAD_NORM = 1 << 28
SENTINEL = np.uint32(0x7F7FFFFF)
INT_MAX = (1 << 31) - 1
RULES = ["lane", "quad", "quad+split", "quad/tile", "union6"]


def chunk_minima(db, qry_block, n_pad):
    """Bracket minima min(||a||^2 - 2 q.a) per (query row, chunk), exact in int64 (the sums are below 2^53)."""
    a = np.zeros((n_pad, db.shape[1]), np.float64)
    a[:len(db)] = db
    na = (a * a).sum(1)
    na[len(db):] = PAD_NORM
    br = na[None, :] - 2.0 * (qry_block.astype(np.float64) @ a.T)
    return br.reshape(len(qry_block), n_pad // CHUNK, CHUNK).min(2).astype(np.int64)


def ceil_f(kmax, keep_mask, chunk_bits):
    """ceil(F) of bracket_bound_not: F = ((kmax & keep_mask) + 2^chunk_bits) as a float, INT_MAX where it is +inf."""
    f = ((kmax & keep_mask) + np.uint32(1 << chunk_bits)).astype(np.uint32).view(np.float32).astype(np.float64)
    return np.where(np.isinf(f), INT_MAX, np.ceil(np.minimum(f, INT_MAX))).astype(np.int64)


def replay_item(M, qn, chunk_bits, rule):
    """M: (256, nchunks) bracket minima, qn: (256,) ||q||^2.  Returns the merged keys (256, 6) and per warp-half
    (passed chunks, network executions, rounds)."""
    rows, nchunks = M.shape
    keep_mask = np.uint32((~((1 << chunk_bits) - 1)) & 0xFFFFFFFF)
    tot = M + qn[:, None]
    keys_all = (tot.astype(np.float64).astype(np.float32).view(np.uint32) & keep_mask) | np.arange(nchunks, dtype=np.uint32)
    S = np.full((rows, 4, NUM_KEYS), SENTINEL, np.uint32)     # [row, lane q, key]
    g4 = np.arange(4)
    passed_l, execs_l, rounds_l = [], [], []
    U = None
    for t in range(nchunks // (TILE // CHUNK)):
        for h in range(2):
            idx = t * 32 + h * 16 + 4 * g4[None, :] + g4[:, None]   # [q, g]
            m, k = tot[:, idx], keys_all[:, idx]                      # [row, q, g]
            if rule == "lane":
                kmax = S[:, :, NUM_KEYS - 1]
            elif rule == "union6":
                kmax = np.repeat(np.sort(S.reshape(rows, -1), 1)[:, NUM_KEYS - 1:NUM_KEYS], 4, 1)
            else:
                if rule != "quad/tile" or h == 0:
                    U = np.minimum(S[:, :, NUM_KEYS - 1].min(1), S[:, :, 1].max(1))
                kmax = np.repeat(U[:, None], 4, 1)
            ok = m < ceil_f(kmax, keep_mask, chunk_bits)[:, :, None]
            p = ok.sum(2).reshape(rows // 16, 2, 8, 4)               # [warp, set, row, lane]
            r = p.max((2, 3))                                          # rounds per warp and set
            joint = r.max(1)
            # round i inserts the lane's i-th chunk in FLO order: passed chunks first, each kind highest g first
            n_rounds = np.repeat(joint[:, None], 2, 1) if rule in ("lane", "quad") else r
            n_rounds = np.repeat(n_rounds, 8, 1).reshape(rows)[:, None, None]
            order = ok * 16 + 4 * g4
            rank = (order[:, :, None, :] > order[:, :, :, None]).sum(3)
            cand = np.where(rank < n_rounds, k, np.uint32(0xFFFFFFFF))
            S = np.sort(np.concatenate([S, cand], 2), 2)[:, :, :NUM_KEYS]
            passed_l.append(p.sum((1, 2, 3)))
            rounds_l.append(joint if rule in ("lane", "quad") else r)
            execs_l.append(2 * joint if rule in ("lane", "quad") else r.sum(1))
    merged = np.sort(S.reshape(rows, -1), 1)[:, :NUM_KEYS]
    assert np.array_equal(merged, np.sort(keys_all, 1)[:, :NUM_KEYS]), "rule %s: the merged keys are not the top 6" % rule
    return np.concatenate(passed_l), np.concatenate(execs_l), np.concatenate([x.ravel() for x in rounds_l])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=4, help="seeded C3 pairs")
    ap.add_argument("--items", type=int, default=3, help="full 256-query items per pair, evenly spaced from the first to the last full one")
    args = ap.parse_args()
    from regard3d_b200 import synth
    sc = synth.make_scene(200, 20000, 128, "sift", seed=20260924 + 3, as_u8=True)   # bench.py's C3 scene
    allp = synth.exhaustive_pairs(200)
    rng = np.random.default_rng(7)
    sel = allp[np.sort(rng.choice(len(allp), args.pairs, replace=False))]
    acc = {r: ([], [], []) for r in RULES}
    for I, J in sel:
        db, qry = sc["descs"][I], sc["descs"][J]
        n_pad = (len(db) + TILE - 1) // TILE * TILE
        nchunks = n_pad // CHUNK
        bits = 4
        while (1 << bits) < nchunks:
            bits += 1
        n_full = len(qry) // ITEM_ROWS     # not the last item: 32 real rows, 224 padding rows that pass almost every bound
        for sb in np.linspace(0, n_full - 1, args.items).round().astype(int):
            blk = np.zeros((ITEM_ROWS, qry.shape[1]), np.int64)
            real = qry[sb * ITEM_ROWS:(sb + 1) * ITEM_ROWS]
            blk[:len(real)] = real
            qn = (blk * blk).sum(1)
            qn[len(real):] = PAD_NORM
            M = chunk_minima(db, blk, n_pad)
            for r in RULES:
                for lst, x in zip(acc[r], replay_item(M, qn, bits, r)):
                    lst.append(x)
        print("pair (%d, %d) done" % (I, J), file=sys.stderr)
    print("%d pairs x %d items, %d warp-halves per rule" % (len(sel), args.items, np.concatenate(acc["lane"][0]).size))
    print("%-11s %8s %8s %9s  %s" % ("rule", "passed", "networks", "rounds", "round histogram 0..4 (per warp and half, or "
                                                                        "per warp, half and set for split loops)"))
    for r in RULES:
        passed, execs, rounds = (np.concatenate(x) for x in acc[r])
        hist = np.bincount(rounds, minlength=5)[:5] / rounds.size * 100
        print("%-11s %8.2f %8.3f %9.3f  %s" % (r, passed.mean(), execs.mean(), rounds.mean(),
                                             " ".join("%5.1f%%" % x for x in hist)))


if __name__ == "__main__":
    main()
