import os
import sys

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import pyoracle
    pyoracle.build()
    return pyoracle


@pytest.fixture(scope="session")
def r3dlib():
    """The product library, built in-tree if needed (nvcc cross-compiles without a GPU)."""
    from regard3d_b200 import build as b
    b.build()
    from regard3d_b200 import capi
    return capi


@pytest.fixture(scope="session")
def gpu_ctx(r3dlib):
    ctx = r3dlib.Context((0,))
    yield ctx
    ctx.close()


def match_sets(ofs, m, pairs):
    out = {}
    for k, (I, J) in enumerate(pairs):
        e = m[int(ofs[k]):int(ofs[k + 1])]
        if len(e):
            out[(int(I), int(J))] = set(zip(e["i"].tolist(), e["j"].tolist()))
    return out


def dict_sets(d):
    return {k: set(zip(v["i"].tolist(), v["j"].tolist())) for k, v in d.items() if len(v)}
