"""r3d_save_features (KeypointSet::saveToBinFile) against the oracle's OpenMVG writers, byte for byte; runs on the
host only."""
import os
import re

import numpy as np
import pytest

NEW_SYMBOLS = ("r3d_extract_default_options", "r3d_extract_features", "r3d_features_descriptors", "r3d_save_features",
               "r3d_get_extract_timing")


def _same_files(tmp_path, a, b):
    for ext in (".feat", ".desc"):
        assert open(str(tmp_path / (a + ext)), "rb").read() == open(str(tmp_path / (b + ext)), "rb").read(), ext


def test_files_equal_oracle_writers(r3dlib, oracle, tmp_path):
    rng = np.random.default_rng(3)
    special = np.float32([1e-5, 12345.67, 4095.5, 0.0, -0.0, 1.0 / 3.0, 359.99997, 1e7, 123456.7, 2.5e-7])
    x = np.concatenate([special, rng.uniform(0, 4000, 200).astype(np.float32)])
    xyso = np.stack([x, np.roll(x, 1), np.abs(np.roll(x, 2)) / np.float32(7), rng.uniform(0, 360, len(x))], 1)
    xyso = xyso.astype(np.float32)
    desc = rng.random((len(x), 144)).astype(np.float32)
    r3dlib.save_features(str(tmp_path / "a.feat"), str(tmp_path / "a.desc"), xyso, desc)
    assert oracle.save_feat(str(tmp_path / "b.feat"), xyso) == 0
    assert oracle.save_desc(str(tmp_path / "b.desc"), desc) == 0
    _same_files(tmp_path, "a", "b")
    lines = open(str(tmp_path / "a.feat")).read().splitlines()
    assert len(lines) == len(x)
    assert [l.split()[0] for l in lines[:4]] == ["1e-05", "12345.7", "4095.5", "0"]  # 6 significant digits
    assert os.path.getsize(str(tmp_path / "a.desc")) == 8 + len(x) * 144 * 4


def test_keypoint_records_write_scale_as_half_size(r3dlib, oracle, tmp_path):
    k = np.zeros(3, r3dlib.akaze_keypoint_dtype)
    k["x"], k["y"], k["size"], k["angle"] = [10.5, 20.25, 4095.5], [1.0, 2.0, 3.0], [9.6, 19.2, 38.4], [0.0, 90.5, 359.5]
    d = np.ones((3, 144), np.float32)
    r3dlib.save_features(str(tmp_path / "a.feat"), str(tmp_path / "a.desc"), k, d)
    xyso = np.stack([k["x"], k["y"], k["size"] / np.float32(2), k["angle"]], 1).astype(np.float32)
    assert oracle.save_feat(str(tmp_path / "b.feat"), xyso) == 0
    assert oracle.save_desc(str(tmp_path / "b.desc"), d) == 0
    _same_files(tmp_path, "a", "b")


def test_zero_keypoints(r3dlib, oracle, tmp_path):
    r3dlib.save_features(str(tmp_path / "a.feat"), str(tmp_path / "a.desc"), np.zeros((0, 4), np.float32),
                         np.zeros((0, 144), np.float32))
    assert oracle.save_feat(str(tmp_path / "b.feat"), np.zeros((0, 4), np.float32)) == 0
    assert oracle.save_desc(str(tmp_path / "b.desc"), np.zeros((0, 144), np.float32)) == 0
    _same_files(tmp_path, "a", "b")
    assert os.path.getsize(str(tmp_path / "a.feat")) == 0 and os.path.getsize(str(tmp_path / "a.desc")) == 8


def test_unwritable_path_is_an_io_error(r3dlib, tmp_path):
    bad = str(tmp_path / "no_such_dir" / "a.feat")
    with pytest.raises(r3dlib.R3DError) as e:
        r3dlib.save_features(bad, str(tmp_path / "a.desc"), np.zeros((1, 4), np.float32), np.zeros((1, 144), np.float32))
    assert e.value.code == -4 and bad in str(e.value)
    bad = str(tmp_path / "no_such_dir" / "a.desc")
    with pytest.raises(r3dlib.R3DError) as e:
        r3dlib.save_features(str(tmp_path / "a.feat"), bad, np.zeros((1, 4), np.float32), np.zeros((1, 144), np.float32))
    assert e.value.code == -4 and bad in str(e.value)


def test_new_symbols_declared_and_exported(r3dlib):
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "r3dgpu.h")).read()
    lib = r3dlib.lib()
    for s in NEW_SYMBOLS:
        assert re.search(r"\b%s\s*\(" % s, header), s
        assert s in r3dlib.EXPORTS and hasattr(lib, s), s
    for t in ("r3d_extract_options", "r3d_extract_timing"):
        assert re.search(r"\}\s*%s;" % t, header), t
    assert hasattr(lib, "r3d_shim_extract_features")
    o = r3dlib.ExtractOptions()
    lib.r3d_extract_default_options(r3dlib.C.byref(o))
    assert o.kp_size_factor == 8.0 and o.out_dir is None and abs(o.akaze.threshold - 1e-3) < 1e-9
    assert o.akaze.octaves == 4 and o.akaze.sublevels == 4
