"""CPU: planarslam_b200/csrc/lsd_rectenum.h - the row-span code the CUDA NFA validation uses for the OpenCV 4.x rectangle
enumeration (pslam_lsd_set_rect_enumeration(ctx, 1)) - compiled for the HOST with g++ and compared with the oracle's statement
of the same enumeration (oracle/lsd.cc rect_rows_cv4, itself pinned against cv2 4.13 by tests/test_oracle_lsd.py).  The header
is plain double arithmetic (nvcc builds it with --fmad=false), so host spans = device spans; the device-side pixel loop is the
same as the validated one of the published iterator; tests/test_lsd_gpu.py runs the device side against the oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("rectenum") / "librectenum_host.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                    "-I", os.path.join(ROOT, "planarslam_b200", "csrc"), "-o", str(out),
                    os.path.join(ROOT, "tests", "host_harness", "lsd_rectenum_host.cc")], check=True)
    L = C.CDLL(str(out))
    L.host_lsd_cv4_spans.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int]
    return L


def _spans(fn, rect, W, H, cap=2048):
    rows = np.zeros((cap, 3), np.int32)
    r = np.ascontiguousarray(rect, np.float64)
    m = fn(r.ctypes.data, W, H, rows.ctypes.data, cap)
    assert m <= cap
    return rows[:m].copy()


def _rect(cx, cy, theta, length, width):
    dx, dy = np.cos(theta), np.sin(theta)
    return [cx - dx * length / 2, cy - dy * length / 2, cx + dx * length / 2, cy + dy * length / 2, width, dx, dy]


def test_rectenum_header_matches_oracle(host_lib):
    O = oracle_lib.lib()
    O.orc_lsd_cv4_spans.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int]
    W, H = 512, 384
    rng = np.random.default_rng(5)
    rects = []
    for _ in range(20000):                                                     # generic rectangles, some leaving the image
        rects.append(_rect(rng.uniform(-20, W + 20), rng.uniform(-20, H + 20), rng.uniform(-np.pi, np.pi), rng.uniform(1, 300), rng.uniform(0.5, 12)))
    for th in np.arange(-4, 5) * (np.pi / 4):                                  # axis-aligned / diagonal, integer and half-integer corners
        for cx, cy in ((100.0, 100.0), (100.5, 77.5), (0.0, 0.0), (W - 1.0, H - 1.0), (255.25, 191.75)):
            for ln, wd in ((40.0, 3.0), (41.0, 4.0), (1.0, 1.0), (600.0, 2.0), (7.0, 0.5)):
                rects.append(_rect(cx, cy, th, ln, wd))
                r = _rect(cx, cy, th, ln, wd)
                r[5], r[6] = float(np.round(r[5])), float(np.round(r[6]))      # exact 0 / +-1 axes: ties between corner rows and columns
                rects.append(r)
    for _ in range(2000):                                                      # corners within an ulp or so of integer rows
        r = _rect(rng.integers(10, W - 10), rng.integers(10, H - 10), rng.choice([0.0, np.pi / 2, np.pi, -np.pi / 2]) + rng.uniform(-1e-12, 1e-12),
                  float(rng.integers(2, 60)), float(rng.integers(1, 8)))
        rects.append(r)
    total = 0
    for r in rects:
        a = _spans(host_lib.host_lsd_cv4_spans, r, W, H)
        b = _spans(O.orc_lsd_cv4_spans, r, W, H)
        assert a.shape == b.shape and np.array_equal(a, b), r
        total += len(a)
    assert total > 200000


def test_rectenum_counts_match_cv2_on_known_rectangle(host_lib):
    """One rectangle measured on cv2 4.13 itself (x ~ 266, y ~ 191..199 of a 512 x 384 level-line field): 23 or 24 points depending
    on the last ulp of the axes; the spans of the header add up to the oracle's count."""
    r = [265.96121405450043, 190.80362514778702, 264.39754256963539, 199.0751525024946, 2.7082036974740857, -0.18575265690440937, 0.98259653492822419]
    a = _spans(host_lib.host_lsd_cv4_spans, r, 512, 384)
    assert int((a[:, 2] - a[:, 1] + 1).sum()) == 24
    assert a[0, 0] == 191 and a[-1, 0] == 199                                 # row 200 (ceil of the bottom corner) is visited but empty


def test_detsincos_header_matches_oracle(host_lib):
    """planarslam_b200/csrc/lsd_detsincos.h compiled for the host == oracle/detmath.h bit for bit: the seed (cos, sin) table of k_lsd_regions is built from it on
    the host, the rectangle axes use it on the device.  Inputs: every angle the detector can produce for a gradient (degrees as float, times pi / 180) plus
    rectangle-axis angles up to 3 pi."""
    import ctypes as C
    import oracle_lib
    host_lib.host_lsd_sincos.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L = oracle_lib.lib()
    L.orc_det_sincos.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    rng = np.random.default_rng(5)
    deg = np.concatenate([rng.uniform(0, 360, 200000).astype(np.float32), np.arange(0, 360, 0.25, dtype=np.float32)])
    x = np.concatenate([deg.astype(np.float64) * 0.0174532925199432957692, rng.uniform(-3 * np.pi, 3 * np.pi, 100000), [0.0, np.pi / 2, np.pi, 2 * np.pi, -np.pi / 2]])
    x = np.ascontiguousarray(x)
    hs, hc, os_, oc = (np.zeros(len(x)) for _ in range(4))
    host_lib.host_lsd_sincos(x.ctypes.data, len(x), hs.ctypes.data, hc.ctypes.data)
    L.orc_det_sincos(x.ctypes.data, len(x), os_.ctypes.data, oc.ctypes.data)
    assert np.array_equal(hs.view(np.uint64), os_.view(np.uint64)) and np.array_equal(hc.view(np.uint64), oc.view(np.uint64))
    assert np.abs(hs - np.sin(x)).max() < 3e-16 and np.abs(hc - np.cos(x)).max() < 3e-16
