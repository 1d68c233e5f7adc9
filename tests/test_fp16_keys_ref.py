"""The float64 reference of the fp16 candidate path (tests/fp16_keys_ref.py) on hand-worked rows: no GPU needed."""
import numpy as np

import fp16_keys_ref as ref


def _row(*vals, dim=16):
    a = np.zeros((1, dim), np.float32)
    a[0, :len(vals)] = vals
    return a


def test_layout_constants():
    assert (ref.kmain(16), ref.operand_cols(16), ref.k16_steps(16)) == (16, 64, 2)
    assert (ref.kmain(17), ref.operand_cols(17), ref.k16_steps(17)) == (32, 64, 3)
    assert (ref.kmain(144), ref.operand_cols(144), ref.k16_steps(144)) == (144, 192, 10)
    assert (ref.kmain(240), ref.operand_cols(240), ref.k16_steps(240)) == (240, 256, 16)
    assert [ref.chunk_bits(n) for n in (2, 256, 257, 2048, 5000)] == [5, 5, 6, 8, 10]
    assert ref.n_pad(0) == ref.n_pad(1) == ref.n_pad(256) == 256 and ref.n_pad(257) == 512


def test_normal_row_splits_exactly():
    # ||a||^2 = 1 + 2^-24, e0 = 0: p0 = 1, remainder 2^-24 = p1 * 2^-11 with p1 = 2^-13 (a normal half)
    a = _row(1.0, 2.0 ** -12)
    n2 = ref.kernel_norm2(a, 16)
    assert n2[0] == 1.0 + 2.0 ** -24
    p0, p1 = ref.norm_split(n2, 0)
    assert (p0[0], p1[0]) == (np.float16(1.0), np.float16(2.0 ** -13))
    assert ref.split_value(p0, p1, 0)[0] == n2[0]
    opQ, opD = ref.prepare(a, 0)
    assert opQ.shape == opD.shape == (256, 64)
    assert list(opD[0, :3]) == [1.0, np.float16(2.0 ** -12), 0.0] and list(opQ[0, :2]) == [-2.0, np.float16(-2.0 ** -11)]
    assert list(opD[0, 16:21]) == [1.0, np.float16(2.0 ** -13), 1.0, np.float16(2.0 ** -11), 0.0]
    assert list(opQ[0, 16:21]) == [1.0, np.float16(2.0 ** -11), 1.0, np.float16(2.0 ** -13), 0.0]
    # the surrogate of a row against itself: ||a||^2 + ||a||^2 - 2 ||a||^2 = 0
    assert ref.surrogate(opQ[:1], opD[:1])[0, 0] == 0.0


def test_subnormal_row_loses_the_low_bits():
    # e0 = 15 (a view with ||a||^2 near 2^28 shares the device): ||a||^2 = 2^-10 + 2^-12 + 2^-26.
    # p0 = fp16(5 * 2^-27) = 2^-24 (subnormal), remainder -3 * 2^-12 + 2^-26; / 2^4 = -3 * 2^-16 + 2^-30, and the
    # subnormal spacing 2^-24 drops the 2^-30: the split is 2^-26 short, within the floor 2^(e0 - 36) = 2^-21
    a = _row(2.0 ** -5, 2.0 ** -6, 2.0 ** -13)
    n2 = ref.kernel_norm2(a, 16)
    assert n2[0] == 2.0 ** -10 + 2.0 ** -12 + 2.0 ** -26
    p0, p1 = ref.norm_split(n2, 15)
    assert (p0[0], p1[0]) == (np.float16(2.0 ** -24), np.float16(-3 * 2.0 ** -16))
    err = n2[0] - ref.split_value(p0, p1, 15)[0]
    assert err == 2.0 ** -26
    assert err > 2.0 ** -21 * n2[0]             # far beyond the relative split term alone
    assert err <= 2.0 ** (15 - 36)


def test_zero_and_padding_rows():
    a = np.zeros((3, 20), np.float32)
    opQ, opD = ref.prepare(a, -3)
    assert ref.kernel_norm2(a, 32).tolist() == [0.0, 0.0, 0.0]
    assert not opQ[:3, :32].any() and not opD[:3, :32].any()
    assert (opQ[:3, :32].view(np.uint16) == 0x8000).all()     # fp16(-2 * 0) = -0, as the kernel writes it
    assert opD[0, 32:36].tolist() == [0.0, 0.0, 0.125, 2.0 ** -14] and opQ[0, 32:36].tolist() == [0.125, 2.0 ** -14, 0.0, 0.0]
    # padding row 3: opQ zero, opD = [0.. | 65504 0 S0 S1 0..]
    assert not opQ[3].view(np.uint16).any()
    assert opD[3, 32:36].tolist() == [65504.0, 0.0, 0.125, 2.0 ** -14] and not opD[3, :32].any() and not opD[3, 36:].any()
    # a padding row's surrogate is 65504 S0 + ||b||^2: above every real distance
    b = _row(3.0, 4.0, dim=20)
    qQ, _ = ref.prepare(b, -3)
    assert ref.surrogate(qQ[:1], opD[3:4])[0, 0] == 65504.0 * 0.125 + 25.0


def test_kernel_norm_order_is_lanes_then_butterfly():
    # 64 columns: lane l holds a_l^2 + a_(l+32)^2; values chosen so that float64 order matters
    a = np.zeros((1, 64), np.float32)
    a[0, 0], a[0, 32], a[0, 16] = 2.0 ** 20, 1.0, 2.0 ** -10
    lane = np.zeros(32)
    lane[0] = np.float64(2.0 ** 40) + 1.0
    lane[16] = 2.0 ** -20
    for o in (16, 8, 4, 2, 1):
        lane = lane + lane[np.arange(32) ^ o]
    assert ref.kernel_norm2(a, 64)[0] == lane[0]


def test_eps_pair_hand_case():
    # database: max||a|| = 2, max||fp16(a)|| = 2, max||a - fp16(a)|| = 2^-12; query: 1, 1, 0; e0 = 3
    sI = np.array([4.0, 4.0, 2.0 ** -24, 1.0])
    sJ = np.array([1.0, 1.0, 0.0, 1.0])
    quant, split, acc = ref.eps_terms(sI, sJ, 3, 64)
    assert quant == 2.0 * (2.0 ** -12 * 1.0 + 2.0 * 0.0)
    assert split == 5.0 * 2.0 ** -21 + 2.0 ** -32
    assert acc == 9.0 * 2.0 ** -18                       # 5 k16 steps: the floor of 8 steps
    assert ref.eps_pair(sI, sJ, 3, 64) == quant + split + acc
    assert ref.eps_terms(sI, sJ, 3, 240)[2] == 9.0 * 16 * 2.0 ** -21   # 16 k16 steps


def test_view_stats_and_chunk_minima():
    a = np.array([[1.0, 2.0 ** -13 + 2.0 ** -25], [0.5, 0.0]], np.float32)   # row 0 is not exact in fp16
    s = ref.view_stats(a)
    h1 = np.float64(np.float16(2.0 ** -13 + 2.0 ** -25))
    assert s[0] == 1.0 + (2.0 ** -13 + 2.0 ** -25) ** 2 and s[1] == 1.0 + h1 ** 2 and s[3] == 1.0
    assert s[2] == (2.0 ** -13 + 2.0 ** -25 - h1) ** 2
    D = np.arange(2 * 10, dtype=np.float64).reshape(2, 10)[:, ::-1]
    cm = ref.chunk_minima(D, 10)
    assert cm.shape == (2, 32) and cm[0, 0] == 2.0 and cm[0, 1] == 0.0 and np.isinf(cm[:, 2:]).all()


def test_unpack_keys():
    k = np.array([np.float32(3.0).view(np.uint32) | 5], np.uint32)
    kv, masked, cid = ref.unpack_keys(k, 4)
    assert masked[0] == 3.0 and cid[0] == 5 and kv[0] == float(np.uint32(k[0]).view(np.float32))
