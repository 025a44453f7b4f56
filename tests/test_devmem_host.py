"""CPU: planarslam_b200/csrc/devmem.h - the owning device / page-locked arrays and the staging slabs of the host-pointer entry points - compiled for the
HOST with g++ against the CUDA runtime.  Checks the slab layout and the state a failed allocation leaves behind: every request made here is one no device
can satisfy (2^60 bytes), so the checks run, and fail the same way, with or without a GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
PSLAM_OK, PSLAM_E_CUDA = 0, -3
HUGE = 1 << 60


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("devmem") / "libdevmem_host.so"
    lib64 = os.path.join(CUDA, "lib64")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-I", os.path.join(ROOT, "planarslam_b200", "csrc"),
                    "-I", os.path.join(CUDA, "include"), "-o", str(out), os.path.join(ROOT, "tests", "host_harness", "devmem_host.cc"),
                    "-L", lib64, "-Wl,-rpath," + lib64, "-lcudart"], check=True)
    L = C.CDLL(str(out))
    L.host_slab_layout.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.host_slab_layout.restype = C.c_long
    L.host_reserve_twice.argtypes = [C.c_int, C.c_int, C.c_ulonglong, C.c_void_p]
    L.host_slab_alloc.argtypes = [C.c_int, C.c_ulonglong, C.POINTER(C.c_int), C.POINTER(C.c_longlong)]
    return L


def _layout(L, elem, counts):
    elem = np.ascontiguousarray(elem, np.int32)
    counts = np.ascontiguousarray(counts, np.int64)
    off = np.zeros(len(elem), np.int64)
    total = L.host_slab_layout(len(elem), elem.ctypes.data, counts.ctypes.data, off.ctypes.data)
    return off, total


def test_slab_segments_are_256_byte_aligned_and_disjoint(host_lib):
    rng = np.random.default_rng(5)
    elem = rng.choice([1, 2, 4, 8, 16, 28], 40)
    counts = rng.integers(0, 5000, 40)
    counts[::7] = 0
    off, total = _layout(host_lib, elem, counts)
    bytes_ = elem.astype(np.int64) * counts
    assert (off % 256 == 0).all()
    assert off[0] == 0
    assert (off[1:] >= off[:-1] + bytes_[:-1]).all()          # no overlap
    assert total == off[-1] + (bytes_[-1] + 255) // 256 * 256 and total % 256 == 0
    assert ((off[1:] - off[:-1]) == (bytes_[:-1] + 255) // 256 * 256).all()      # no padding beyond the alignment


def test_slab_zero_length_segments(host_lib):
    off, total = _layout(host_lib, [4, 8, 1, 16], [0, 0, 3, 0])
    assert list(off) == [0, 0, 0, 256] and total == 256
    off, total = _layout(host_lib, [2], [0])
    assert list(off) == [0] and total == 0
    off, total = _layout(host_lib, [1, 1], [256, 257])
    assert list(off) == [0, 256] and total == 768


@pytest.mark.parametrize("pinned", [0, 1])
@pytest.mark.parametrize("slack", [0, 1])
def test_failed_reserve_leaves_the_array_empty(host_lib, pinned, slack):
    """A request no device can satisfy returns PSLAM_E_CUDA and leaves null / cap 0; the next request tries again and fails the same way (nothing is
    kept from the failed attempt, so nothing leaks and no freed pointer survives)."""
    st = np.full(6, 7, np.int64)
    host_lib.host_reserve_twice(pinned, slack, HUGE, st.ctypes.data)
    assert list(st) == [PSLAM_E_CUDA, 0, 0, PSLAM_E_CUDA, 0, 0]


def test_reserve_within_capacity_keeps_the_block(host_lib):
    assert host_lib.host_reserve_within_cap() == 1


@pytest.mark.parametrize("ctx", [0, 1])
def test_failed_slab_alloc(host_lib, ctx):
    base_null, cap = C.c_int(0), C.c_longlong(7)
    assert host_lib.host_slab_alloc(ctx, HUGE, C.byref(base_null), C.byref(cap)) == PSLAM_E_CUDA
    assert base_null.value == 1 and cap.value == 0
