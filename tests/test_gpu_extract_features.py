"""-m gpu: r3d_extract_features -- Fast-AKAZE keypoints described with LIOP on the resident images, written as
.feat / .desc -- against the CPU reference composed from the oracle (tests/features_ref.py), byte for byte; then the
whole compute-matches stage from decoded gray images to matches.f.txt."""
import ctypes as C
import os

import numpy as np
import pytest

import features_ref as fr
from akaze_scenes import scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from regard3d_b200 import capi
    c = capi.Context((0,))
    yield c
    c.close()


def _files(d, name):
    return tuple(open(os.path.join(str(d), name + ext), "rb").read() for ext in (".feat", ".desc"))


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _same_arrays(a, b):
    assert a[0].tobytes() == b[0].tobytes(), "keypoints differ"
    assert np.array_equal(_bits(a[1]), _bits(b[1])), "descriptors differ"


@pytest.mark.parametrize("kind,w,h,threshold", [
    ("scene", 641, 479, 1e-3),    # odd sides
    ("scene", 640, 480, 1e-4),    # a second threshold
    ("scene", 150, 120, 1e-4),    # one octave
    ("scene", 4000, 3000, 1e-3),
    ("blank", 320, 240, 1e-3),
    ("constant", 320, 240, 1e-3),
    ("scene", 59, 200, 1e-3),     # too small for one level: empty .feat, 8-byte .desc
])
def test_files_equal_reference(ctx, tmp_path, kind, w, h, threshold):
    img = scene(w, h, seed=w + h) if kind == "scene" else np.full((h, w), 0.0 if kind == "blank" else 0.5, np.float32)
    gpu, ref = tmp_path / "gpu", tmp_path / "ref"
    gpu.mkdir()
    ref.mkdir()
    got = ctx.extract_features([img], out_dir=str(gpu), basenames=["image000000"], threshold=threshold)[0]
    exp = fr.extract_to(ref, [img], ["image000000"], threshold)[0]
    _same_arrays(got, exp)
    assert _files(gpu, "image000000") == _files(ref, "image000000")
    if kind != "scene" or w == 59:
        assert len(got[0]) == 0 and os.path.getsize(str(gpu / "image000000.desc")) == 8
    else:
        assert len(got[0]) > 0


def _mixed_images():
    sizes = [(640, 480), (641, 479), (320, 240), (150, 120), (59, 200), (400, 300), (333, 222)]
    return [scene(*sizes[k % len(sizes)], seed=100 + k) for k in range(20)]


def test_batches_equal_single_calls_and_existing_calls(ctx, tmp_path):
    imgs = _mixed_images()
    names = ["image%06d" % k for k in range(len(imgs))]
    seen = []
    batch = ctx.extract_features(imgs, out_dir=str(tmp_path), basenames=names, threshold=1e-4,
                                 progress=lambda f, m, u: seen.append(f))
    t = ctx.extract_timing()
    assert t["images"] == 20 and t["batches"] >= 2 and t["devices"] == 1
    assert t["keypoints"] == sum(len(k) for k, _ in batch) and t["describe_ms"] > 0
    # progress: one call per image, 0.2 + 0.4 / n up to 0.6, never decreasing
    n = len(imgs)
    assert len(seen) == n and all(b >= a for a, b in zip(seen, seen[1:]))
    assert seen[0] == pytest.approx(0.2 + 0.4 / n, abs=1e-6) and seen[-1] == pytest.approx(0.6, abs=1e-6)
    again = ctx.extract_features(imgs, threshold=1e-4)
    dets = ctx.akaze_detect(imgs, threshold=1e-4)
    for k, img in enumerate(imgs):
        one_dir = tmp_path / ("one%d" % k)
        one_dir.mkdir()
        one = ctx.extract_features([img], out_dir=str(one_dir), basenames=[names[k]], threshold=1e-4)[0]
        _same_arrays(batch[k], one)
        _same_arrays(batch[k], again[k])
        assert _files(tmp_path, names[k]) == _files(one_dir, names[k])
        # the existing calls: r3d_akaze_detect's keypoints, r3d_liop_describe's descriptors of them
        kp = batch[k][0]
        assert kp.tobytes() == dets[k].tobytes()
        k4 = np.stack([kp["x"], kp["y"], kp["size"], kp["angle"]], 1)
        assert np.array_equal(_bits(ctx.liop_describe(img, k4, 8.0)), _bits(batch[k][1]))
    assert sum(len(b[0]) > 0 for b in batch) >= 15


def test_invalid_inputs_write_nothing(ctx, tmp_path):
    from regard3d_b200 import capi
    good = scene(200, 150, seed=1)
    nan = scene(200, 150, seed=2)
    nan[7, 9] = np.nan
    cases = [
        dict(images=[good, nan], basenames=["a", "b"]),                         # a non-finite pixel
        dict(images=[good, np.zeros((2, 50), np.float32)], basenames=["a", "b"]),  # a side <= 2
        dict(images=[good, np.zeros((50, 2), np.float32)], basenames=["a", "b"]),
        dict(images=[good, good], basenames=None),                               # no basenames
        dict(images=[good, good], basenames=["a", ""]),                          # an empty basename
    ]
    for c in cases:
        with pytest.raises(capi.R3DError) as e:
            ctx.extract_features(c["images"], out_dir=str(tmp_path), basenames=c["basenames"])
        assert e.value.code == -1
        assert os.listdir(str(tmp_path)) == []
    with pytest.raises(capi.R3DError) as e:
        ctx.extract_features([good], out_dir="", basenames=["a"])
    assert e.value.code == -1
    with pytest.raises(capi.R3DError) as e:
        ctx.extract_features([good], kp_size_factor=float("nan"))
    assert e.value.code == -1


def test_unwritable_directory_is_an_io_error(ctx, tmp_path):
    from regard3d_b200 import capi
    bad = str(tmp_path / "missing")
    with pytest.raises(capi.R3DError) as e:
        ctx.extract_features([scene(200, 150, seed=1)], out_dir=bad, basenames=["a"])
    assert e.value.code == -4 and bad in str(e.value)


def _crops():
    """Four overlapping 960 x 720 crops of one 1280 x 960 scene at known offsets."""
    big = scene(1280, 960, seed=11)
    offs = [(0, 0), (320, 0), (0, 240), (280, 200)]
    return [np.ascontiguousarray(big[y:y + 720, x:x + 960]) for x, y in offs], offs


def _read_matches(path):
    out, tok = {}, open(path).read().split()
    k = 0
    while k < len(tok):
        I, J, n = int(tok[k]), int(tok[k + 1]), int(tok[k + 2])
        k += 3
        out[(I, J)] = np.array(tok[k:k + 2 * n], np.int64).reshape(n, 2)
        k += 2 * n
    return out


def test_end_to_end_crops(ctx, oracle, tmp_path):
    from regard3d_b200 import synth
    imgs, offs = _crops()
    names = ["image%06d" % v for v in range(len(imgs))]
    gpu, ref = tmp_path / "gpu", tmp_path / "ref"
    gpu.mkdir()
    ref.mkdir()
    ctx.extract_features(imgs, out_dir=str(gpu), basenames=names)
    fr.extract_to(ref, imgs, names)
    for nm in names:
        assert _files(gpu, nm) == _files(ref, nm)
    ws, hs = [960] * 4, [720] * 4
    ctx.compute_matches(str(gpu), names, ws, hs, dist_ratio=0.6, dim=144)
    # the oracle's matcher and F filter on the reference's files
    xys = [oracle.load_feat(str(ref / (nm + ".feat")))[:, :2].copy() for nm in names]
    descs = [oracle.load_desc(str(ref / (nm + ".desc")), 144) for nm in names]
    pairs = synth.exhaustive_pairs(4)
    ofs, m = oracle.match_pairs(descs, xys, pairs, 0.6)
    fo, fm = oracle.filter_pairs_F(xys, ws, hs, pairs, ofs, m)
    oracle.save_matches_txt(str(tmp_path / "put.txt"), pairs, ofs, m)
    oracle.save_matches_txt(str(tmp_path / "f.txt"), pairs, fo, fm)
    assert open(str(gpu / "matches.putative.txt")).read() == open(str(tmp_path / "put.txt")).read()
    assert open(str(gpu / "matches.f.txt")).read() == open(str(tmp_path / "f.txt")).read()
    # the F inliers agree with the known offsets
    good = total = 0
    for (I, J), ij in _read_matches(str(gpu / "matches.f.txt")).items():
        pI = xys[I][ij[:, 0]] + np.float32(offs[I])
        pJ = xys[J][ij[:, 1]] + np.float32(offs[J])
        good += int((np.linalg.norm(pI - pJ, axis=1) <= 2.0).sum())
        total += len(ij)
    assert total >= 100 and good >= 0.8 * total, (good, total)


def test_shim_extract_then_compute_matches(r3dlib, ctx, tmp_path):
    imgs, _ = _crops()
    lib = r3dlib.lib()
    n = len(imgs)
    files = (C.c_char_p * n)(*[("image%06d.jpg" % v).encode() for v in range(n)])
    ptrs = (C.c_void_p * n)(*[im.ctypes.data for im in imgs])
    w = (C.c_uint32 * n)(*[960] * n)
    h = (C.c_uint32 * n)(*[720] * n)
    kp = (C.c_uint32 * n)()
    last = C.c_float()
    rc = lib.r3d_shim_extract_features(str(tmp_path).encode(), files, ptrs, w, h, n, C.c_float(1e-3), None, kp,
                                       C.byref(last))
    assert rc == 0 and last.value == pytest.approx(0.6, abs=1e-6)
    exp = ctx.extract_features(imgs)
    assert list(kp) == [len(k) for k, _ in exp] and min(kp) > 0
    kp2 = (C.c_uint32 * n)()
    pp, fp = C.c_uint64(), C.c_uint64()
    rc = lib.r3d_shim_compute_matches(str(tmp_path).encode(), files, w, h, n, C.c_float(0.6), 4, kp2, C.byref(pp),
                                      C.byref(fp), C.byref(last))
    assert rc == 0 and list(kp2) == list(kp) and pp.value > 0 and fp.value > 0
    other = tmp_path / "other"
    other.mkdir()
    rc = lib.r3d_shim_extract_features(str(other).encode(), files, ptrs, w, h, n, C.c_float(1e-3), b"AKAZE", kp,
                                       C.byref(last))
    assert rc == -1 and os.listdir(str(other)) == []


def test_two_devices_equal_one(tmp_path):
    import torch
    from regard3d_b200 import capi
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    imgs = _mixed_images()[:7]
    names = ["image%06d" % k for k in range(len(imgs))]
    (tmp_path / "one").mkdir()
    (tmp_path / "two").mkdir()
    c1, c2 = capi.Context((0,)), capi.Context((0, 1))
    try:
        one = c1.extract_features(imgs, out_dir=str(tmp_path / "one"), basenames=names, threshold=1e-4)
        two = c2.extract_features(imgs, out_dir=str(tmp_path / "two"), basenames=names, threshold=1e-4)
        assert c2.extract_timing()["devices"] == 2
        for k in range(len(imgs)):
            _same_arrays(one[k], two[k])
            assert _files(tmp_path / "one", names[k]) == _files(tmp_path / "two", names[k])
    finally:
        c1.close()
        c2.close()
