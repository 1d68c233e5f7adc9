"""The Fast-AKAZE restatement (oracle/oracle_akaze.cpp) against OpenCV's own primitives (cv2), numpy and plain-Python
restatements of the extrema passes and the orientation.  Bounds are in ulp of the output's maximum magnitude (float32,
2^-23 relative); the measured worst cases are recorded in DESIGN.md section 2."""
import math

import numpy as np
import pytest

from akaze_scenes import scene
from oracle import pyoracle_akaze as pa

cv2 = pytest.importorskip("cv2")


def _ulp_of_max(got, exp):
    return float(np.abs(got.astype(np.float64) - exp).max() / (np.abs(exp).max() * 2.0 ** -23))


@pytest.fixture(scope="module")
def img():
    return scene(131, 97, seed=3)


def test_gaussian_kernels_bit_exact():
    for sigma in (1.0, 1.6, 1.2, 2.5):
        n = int(math.ceil(np.float32(2.0) * (np.float32(1.0) + (np.float32(sigma) - np.float32(0.8)) / np.float32(0.3))))
        n += 1 - n % 2
        s = float(np.float32(sigma))
        exp = cv2.getGaussianKernel(n, s, ktype=cv2.CV_32F).ravel()
        assert np.array_equal(pa.gaussian_kernel(n, s).view(np.uint32), exp.view(np.uint32))


def test_deriv_kernels_bit_exact():
    for dx, dy in ((1, 0), (0, 1)):
        kx, ky = pa.deriv_kernels(dx, dy, 1)
        ex, ey = cv2.getDerivKernels(dx, dy, -1, normalize=True, ktype=cv2.CV_32F)
        assert np.array_equal(kx, ex.ravel()) and np.array_equal(ky, ey.ravel())
    kx, ky = pa.deriv_kernels(1, 0, 3)  # three taps spread over 7: [-1 .. 1] and 3/32, 10/32, 3/32
    assert np.array_equal(kx, np.float32([-1, 0, 0, 0, 0, 0, 1]))
    np.testing.assert_allclose(ky[[0, 3, 6]], [3 / 32, 10 / 32, 3 / 32], rtol=1e-6)


def test_gaussian_blur_replicate(img):
    for sigma, n in ((1.6, 9), (1.0, 5)):
        exp = cv2.GaussianBlur(img, (n, n), float(np.float32(sigma)), borderType=cv2.BORDER_REPLICATE)
        assert _ulp_of_max(pa.gaussian_blur(img, sigma), exp) <= 4


def test_scharr_and_sep_filter_reflect101(img):
    for dx, dy in ((1, 0), (0, 1)):
        assert _ulp_of_max(pa.scharr(img, dx, dy), cv2.Scharr(img, cv2.CV_32F, dx, dy)) <= 16
    for scale in (1, 2, 3, 4):
        for dx, dy in ((1, 0), (0, 1)):
            kx, ky = pa.deriv_kernels(dx, dy, scale)
            assert _ulp_of_max(pa.sep_filter(img, kx, ky), cv2.sepFilter2D(img, cv2.CV_32F, kx, ky)) <= 8


@pytest.mark.parametrize("h,w", [(96, 130), (97, 131), (96, 131), (97, 130)])
def test_halfsample_inter_area(img, h, w):
    src = np.ascontiguousarray(img[:h, :w])
    exp = cv2.resize(src, (w // 2, h // 2), interpolation=cv2.INTER_AREA)
    assert _ulp_of_max(pa.halfsample(src), exp) <= 1


def test_fast_atan2_against_phase():
    rng = np.random.default_rng(1)
    x = rng.normal(size=4000).astype(np.float32)
    y = rng.normal(size=4000).astype(np.float32)
    x[:8] = [0, 0, 1, -1, 0, 1e-30, -2, 3]
    y[:8] = [0, 1, 0, 0, -1, -1e-30, -2, 3]
    exp = cv2.phase(x.reshape(-1, 1), y.reshape(-1, 1)).ravel()
    assert np.abs(pa.fast_atan2(y, x) - exp).max() <= 2 * 2.0 ** -21  # 2 ulp at 2 pi


def test_solve2_against_cv2_solve():
    rng = np.random.default_rng(2)
    for _ in range(500):
        A = rng.normal(size=(2, 2)).astype(np.float32)
        A[1, 0] = A[0, 1]
        b = rng.normal(size=2).astype(np.float32)
        _, exp = cv2.solve(A, b.reshape(2, 1), flags=cv2.DECOMP_LU)
        assert np.array_equal(pa.solve2(A, b), exp.ravel())
    singular = np.float32([[1, 2], [2, 4]])
    ok, exp = cv2.solve(singular, np.float32([[1], [1]]), flags=cv2.DECOMP_LU)
    assert not ok and np.array_equal(pa.solve2(singular, np.float32([1, 1])), exp.ravel())  # zeros


def test_k_percentile_against_numpy(img):
    lx, ly = pa.scharr(img, 1, 0), pa.scharr(img, 0, 1)
    m = np.sqrt(lx[1:-1, 1:-1] ** 2 + ly[1:-1, 1:-1] ** 2).astype(np.float32).ravel()
    hmax = m.max()
    hist = np.bincount((m * (np.float32(299) / hmax)).astype(np.int32), minlength=300)
    nthr = int(np.float32(len(m) - hist[0]) * np.float32(0.7))
    cum = np.concatenate([[0], np.cumsum(hist[1:])])
    k = int(np.argmax(cum >= nthr)) + 1
    assert pa.k_percentile(lx, ly) == np.float32(hmax * np.float32(k)) / np.float32(300)
    z = np.zeros((20, 20), np.float32)
    assert pa.k_percentile(z, z) == np.float32(0.03)


def test_fed_tau_sums_to_the_time_step():
    lv = pa.level_table(640, 480)
    for i in range(1, len(lv)):
        dt = lv["etime"][i] - lv["etime"][i - 1]
        tau = pa.fed_tau(dt)
        assert len(tau) == lv["n_tau"][i] and len(tau) > 0
        assert abs(float(tau.astype(np.float64).sum()) - float(dt)) <= 1e-5 * float(dt)


def test_gauss25_table():
    g = pa.gauss25()
    assert g[0, 0] == np.float32(0.02546481) and g[6, 6] == np.float32(0.00008024) and g[3, 4] == np.float32(0.00344629)


def _plain_passes(levels, threshold):
    """The three extrema passes restated in plain Python (sequential lower and upper passes as upstream runs them)."""
    kpts = []
    for i, d in enumerate(levels):
        L, lv = d["Ldet"], d["level"]
        b, w, h = int(lv["border"]), int(lv["width"]), int(lv["height"])
        size = np.float32(lv["esigma"]) * np.float32(1.5)
        out = []
        for y in range(b, h - b):
            for x in range(b, w - b):
                v = L[y, x]
                if v <= np.float32(threshold):
                    continue
                nb = L[y - 1:y + 2, x - 1:x + 2].ravel()
                if any(v <= nb[k] for k in (0, 1, 2, 3, 5, 6, 7, 8)):
                    continue
                p = [np.float32(x * lv["ratio"]), np.float32(y * lv["ratio"]), size, v]
                for j, q in enumerate(out):
                    dx, dy = p[0] - q[0], p[1] - q[1]
                    if dx * dx + dy * dy <= size * size:
                        if p[3] > q[3]:
                            out[j] = p
                        break
                else:
                    out.append(p)
        kpts.append(out)
    lower = [[False] * len(k) for k in kpts]
    for i in range(1, len(kpts)):
        for p in kpts[i]:
            for j, q in enumerate(kpts[i - 1]):
                if lower[i - 1][j]:
                    continue
                dx, dy = p[0] - q[0], p[1] - q[1]
                if dx * dx + dy * dy <= p[2] * p[2] and p[3] > q[3]:
                    lower[i - 1][j] = True
    upper = [list(f) for f in lower]
    for i in range(len(kpts) - 2, -1, -1):
        for j, p in enumerate(kpts[i]):
            if upper[i][j]:
                continue
            for k, q in enumerate(kpts[i + 1]):
                if upper[i + 1][k]:
                    continue
                dx, dy = p[0] - q[0], p[1] - q[1]
                if dx * dx + dy * dy <= q[2] * q[2] and p[3] > q[3]:
                    upper[i + 1][k] = True
    return kpts, lower, upper


def _parallel_deletions(kpts, lower):
    """Passes 2 and 3 as independent neighbour queries (what the GPU runs): the same flags as the sequential loops."""
    n = len(kpts)
    lo = [[any((p[0] - q[0]) ** 2 + (p[1] - q[1]) ** 2 <= p[2] * p[2] and p[3] > q[3] for p in kpts[i + 1])
           if i + 1 < n else False for q in kpts[i]] for i in range(n)]
    up = [[lo[i][k] or (i > 0 and any(not lo[i - 1][j] and (p[0] - q[0]) ** 2 + (p[1] - q[1]) ** 2 <= q[2] * q[2]
                                      and p[3] > q[3] for j, p in enumerate(kpts[i - 1])))
           for k, q in enumerate(kpts[i])] for i in range(n)]
    return lo, up


def test_extrema_passes_against_plain_python():
    img = scene(200, 160, seed=11, n_shapes=40)
    _, levels, _ = pa.detect(img, 1e-4, levels=True)
    kpts, lower, upper = _plain_passes(levels, 1e-4)
    assert sum(len(k) for k in kpts) > 20
    assert any(any(f) for f in lower) and any(u and not l for U, Lw in zip(upper, lower) for u, l in zip(U, Lw))
    plo, pup = _parallel_deletions(kpts, lower)
    for i, d in enumerate(levels):
        c = d["candidates"]
        assert len(c) == len(kpts[i])
        for j, p in enumerate(kpts[i]):
            assert (c["x"][j], c["y"][j], c["size"][j], c["response"][j]) == tuple(np.float32(v) for v in p)
        assert list(d["deleted_lower"]) == lower[i] == plo[i]
        assert list(d["deleted_upper"]) == upper[i] == pup[i]


def test_orientation_against_numpy():
    img = scene(320, 240, seed=5)
    kps, levels, ori = pa.detect(img, 1e-3, levels=True)
    assert len(kps) > 10
    g = pa.gauss25()
    for kp, (mx, my) in list(zip(kps, ori))[:40]:
        lv = levels[kp["class_id"]]
        ratio = lv["level"]["ratio"]
        scale = int(np.float32(0.5) * kp["size"] / ratio + np.float32(0.5))
        x0, y0 = int(kp["x"] / ratio + np.float32(0.5)), int(kp["y"] / ratio + np.float32(0.5))
        rx, ry = [], []
        for i in range(-6, 7):
            for j in range(-6, 7):
                if i * i + j * j < 36:
                    wgt = g[abs(i), abs(j)]
                    rx.append(wgt * lv["Lx"][y0 + i * scale, x0 + j * scale])
                    ry.append(wgt * lv["Ly"][y0 + i * scale, x0 + j * scale])
        rx, ry = np.float32(rx), np.float32(ry)
        sl = (pa.fast_atan2(ry, rx) / np.float32(2 * np.pi / 42)).astype(int)
        best = None
        for s0 in range(42):  # every 7-slice window, wrapping around
            m = np.isin(sl, [(s0 + k) % 42 for k in range(7)])
            sx, sy = float(rx[m].astype(np.float64).sum()), float(ry[m].astype(np.float64).sum())
            if best is None or sx * sx + sy * sy > best[0]:
                best = (sx * sx + sy * sy, sx, sy)
        # float32 sums in the counting sort's order differ from these in the last bits
        assert abs(mx - best[1]) <= 1e-4 * (abs(best[1]) + abs(best[2])) + 1e-9
        assert abs(my - best[2]) <= 1e-4 * (abs(best[1]) + abs(best[2])) + 1e-9
        a = math.degrees(math.atan2(my, mx)) % 360.0 + 90.0
        a = a - 360.0 if a > 360.0 else a
        assert abs(kp["angle"] - a) <= 1e-3


def test_level_table_640x480_written_out():
    """The level table of a 640x480 image, worked by hand from Allocate_Memory_Evolution: esigma = 1.6 2^(j/4 + i),
    sigma_size = round(1.5 esigma / 2^i) = 2, 3, 3, 4 per sublevel, border = round(10 sqrt(2) sigma_size) + 1 =
    29, 43, 43, 58; octave 3 (80x60) keeps only sublevel 0 (2 * 43 + 1 >= 60).  Both the oracle and the library."""
    from regard3d_b200 import capi
    shapes = [(640, 480)] * 4 + [(320, 240)] * 4 + [(160, 120)] * 4 + [(80, 60)]
    exp_ss, exp_border = [2, 3, 3, 4] * 3 + [2], [29, 43, 43, 58] * 3 + [29]
    for lv in (pa.level_table(640, 480), capi.akaze_levels(640, 480)):
        assert [(int(l["width"]), int(l["height"])) for l in lv] == shapes
        assert list(lv["sigma_size"]) == exp_ss and list(lv["border"]) == exp_border
        assert list(lv["octave"]) == [0] * 4 + [1] * 4 + [2] * 4 + [3]
        np.testing.assert_allclose(lv["esigma"], [1.6 * 2 ** (j / 4 + i) for i in range(4) for j in range(4)][:13],
                                   rtol=1e-6)
        for i in range(1, 13):  # fed_tau_by_cycle_timeV2's step count, n = ceil(sqrt(3 T / 0.25 + 1/4) - 1/2)
            T = (lv["esigma"][i] ** 2 - lv["esigma"][i - 1] ** 2) / 2
            assert lv["n_tau"][i] == math.ceil(math.sqrt(3 * T / 0.25 + 0.25) - 0.5 - 1e-8)


def test_level_table_rules():
    lv = pa.level_table(640, 480)
    assert len(lv) == 13 and lv["octave"][-1] == 3
    assert len(pa.level_table(150, 120)) == 4 and set(pa.level_table(150, 120)["octave"]) == {0}  # next octave < 80
    lv = pa.level_table(100, 100)  # 2 * border + 1 >= side ends the list mid-octave
    assert len(lv) == 3 and 2 * (int(lv["border"][-1])) + 1 < 100
    assert len(pa.level_table(40, 40)) == 0


# overlap floor against cv2.AKAZE_create, a related implementation (not the reference): see DESIGN.md section 2
def test_end_to_end_overlap_with_cv2_akaze():
    img = scene(640, 480, seed=21)
    kps = pa.detect(img, 1e-3)
    det = cv2.AKAZE_create(threshold=1e-3, nOctaves=4, nOctaveLayers=4, diffusivity=cv2.KAZE_DIFF_PM_G2)
    ref = det.detect(img, None)
    assert len(kps) > 50 and len(ref) > 50
    rp = np.float32([k.pt for k in ref])
    d = np.sqrt(((np.stack([kps["x"], kps["y"]], 1)[:, None, :] - rp[None]) ** 2).sum(-1)).min(1)
    overlap = float((d <= 1.5).mean())
    assert overlap >= 0.85, overlap  # measured 0.96-0.97 (1.5 px) on seeds 21-23
