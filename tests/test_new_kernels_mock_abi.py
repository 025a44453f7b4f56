"""CPU: the Python mirrors and the GPU test bodies of the entry points added after the round-1 GPU budget was spent (isLineGood,
TrackManhattanFrame, map-line frustum test, ComputeStereoFromRGBD), run end to end against a CPU stand-in of those entry points.

The stand-in (tests/host_harness/mock_abi.cc) is built from the same shared host/device bodies the CUDA kernels call and includes
include/pslam_abi.h, so its signatures are the real ABI's.  What this covers that the per-body host tests do not: argument order
and dtypes of the ctypes calls, array shapes / padding of the batch forms, and the assertions of the GPU tests themselves - so that
the first run on a GPU can only fail for a reason inside the kernels' launch code.  Test infrastructure only: the product library
is not involved and keeps having no CPU path."""
import ctypes as C
import os
import subprocess
import types

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fake_context(tmp_path_factory):
    out = tmp_path_factory.mktemp("mock") / "libmock_abi.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", os.path.join(ROOT, "planarslam_b200", "csrc"),
                    "-I", os.path.join(ROOT, "include"), "-o", str(out), os.path.join(ROOT, "tests", "host_harness", "mock_abi.cc")], check=True)
    L = C.CDLL(str(out))
    from planarslam_b200 import _lib
    real = _lib.lib()                                     # the product library (loads without a GPU): its argtypes are what the mirrors rely on
    for name in ("pslam_lines3d_batch", "pslam_track_manhattan_batch", "pslam_lines_in_frustum", "pslam_compute_stereo_from_rgbd_batch"):
        getattr(L, name).argtypes = getattr(real, name).argtypes
    L.mock_create.restype = C.c_void_p
    L.mock_create.argtypes = [C.c_int, C.c_int]
    L.pslam_last_error.restype = C.c_char_p

    class FakeContext:
        def __init__(self, width, height, max_batch=1, device=0, **kw):
            self.cfg = types.SimpleNamespace(width=width, height=height, max_batch=max_batch)
            self.L = L
            self.h = C.c_void_p(L.mock_create(width, height))

        def check(self, rc, allow_capacity=False):
            assert rc == 0, rc
            return rc

    return FakeContext


def _run_gpu_test(monkeypatch, fake_context, module_name, test_name):
    import importlib
    from planarslam_b200 import _lib
    monkeypatch.setattr(_lib, "Context", fake_context)
    mod = importlib.import_module(module_name)
    getattr(mod, test_name)()


def test_lines3d_gpu_test_body_on_the_stand_in(monkeypatch, fake_context):
    _run_gpu_test(monkeypatch, fake_context, "test_line3d_gpu", "test_lines3d_match_oracle")


def test_manhattan_gpu_test_body_on_the_stand_in(monkeypatch, fake_context):
    _run_gpu_test(monkeypatch, fake_context, "test_manhattan_gpu", "test_track_manhattan_matches_oracle")


def test_linefrustum_gpu_test_body_on_the_stand_in(monkeypatch, fake_context):
    _run_gpu_test(monkeypatch, fake_context, "test_linefrustum_gpu", "test_lines_in_frustum_match_oracle")


def test_stereo_gpu_test_body_on_the_stand_in(monkeypatch, fake_context):
    _run_gpu_test(monkeypatch, fake_context, "test_framefill", "test_stereo_from_rgbd_gpu_matches_oracle")
