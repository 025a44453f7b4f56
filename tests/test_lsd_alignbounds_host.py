"""CPU: planarslam_b200/csrc/lsd_alignbounds.h - the word intervals the CUDA NFA validation counts aligned pixels with - compiled for the HOST with g++ and
checked against the exact alignment test (lsd_aligned_angle of the word's angle) it replaces.  The header is plain double arithmetic (nvcc builds it with
--fmad=false), so the host bounds are the device bounds; tests/test_lsd_gpu.py runs the device side against the oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNDEF = 0x7F800000


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("alignbounds") / "libalignbounds_host.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                    "-I", os.path.join(ROOT, "planarslam_b200", "csrc"), "-o", str(out),
                    os.path.join(ROOT, "tests", "host_harness", "lsd_alignbounds_host.cc")], check=True)
    L = C.CDLL(str(out))
    L.host_lsd_align_set.argtypes = [C.c_double, C.c_double, C.c_void_p]
    L.host_lsd_align_mismatches.argtypes = [C.c_void_p, C.c_long, C.c_double, C.c_double]
    L.host_lsd_align_mismatches.restype = C.c_long
    return L


@pytest.fixture(scope="module")
def reachable_words():
    """Every angle word k_lsd_gradient can store: cv::fastAtan2(gx, -gy) in degrees for gx, gy in [-510, 510] (the oracle's cv2-pinned fastAtan2),
    with and without the used bit, plus the undefined word and NaN words."""
    L = oracle_lib.lib()
    fa = L.orc_fast_atan2
    deg = np.array([fa(float(gx), float(-gy)) for gx in range(-510, 511) for gy in range(-510, 511)], np.float32)
    w = np.unique(deg.view(np.uint32))
    assert len(w) > 100000 and w.max() < UNDEF
    w = np.concatenate([w, w | 0x80000000, [UNDEF, UNDEF | 0x80000000, UNDEF + 1, 0x7FFFFFFF]]).astype(np.uint32)
    return np.ascontiguousarray(w)


def _precs():
    return [0.125 * 2.0 ** -j * np.pi for j in range(11)]


def _check(L, w, thetas):
    bad = []
    for th in thetas:
        for prec in _precs():
            m = L.host_lsd_align_mismatches(w.ctypes.data, len(w), float(th), float(prec))
            if m:
                bad.append((float(th), prec, m))
    assert not bad, bad[:5]


def test_alignbounds_random_angles(host_lib, reachable_words):
    rng = np.random.default_rng(7)
    _check(host_lib, reachable_words, rng.uniform(-np.pi, 3 * np.pi, 40))


def test_alignbounds_edge_angles(host_lib, reachable_words):
    """theta near 0, +-pi, 2 pi and 3 pi, and where theta - a crosses the 3 pi / 2 switch or the wrap-around window edges (2 pi +- prec)."""
    base = [0.0, np.pi, -np.pi, 2 * np.pi, 3 * np.pi, np.pi / 2, 1.5 * np.pi, -1.5 * np.pi, 5 * np.pi / 4]
    for prec in _precs():
        base += [2 * np.pi - prec, 2 * np.pi + prec, prec, -prec, np.pi + prec, 1.5 * np.pi + prec, 1.5 * np.pi - prec]
    thetas = []
    for t in base:
        thetas += [t, np.nextafter(t, np.inf), np.nextafter(t, -np.inf), t + 1e-9, t - 1e-9]
    _check(host_lib, reachable_words, thetas)


def test_alignbounds_detector_angles(host_lib, reachable_words):
    """Rectangle angles as the detector forms them: an angle word's own angle, and that angle + pi (region2rect flips theta by pi)."""
    rng = np.random.default_rng(3)
    w = rng.choice(reachable_words[reachable_words < UNDEF], 20)
    a = w.view(np.float32).astype(np.float64) * (np.pi / 180)
    _check(host_lib, reachable_words, np.concatenate([a, a + np.pi]))


def test_alignbounds_intervals_shape(host_lib):
    """The set around theta is never empty for a theta inside the angle range, and all intervals stay below the undefined word."""
    out = np.zeros(6, np.uint32)
    for th in np.linspace(0.01, 2 * np.pi - 0.01, 50):
        for prec in _precs():
            host_lib.host_lsd_align_set(float(th), float(prec), out.ctypes.data)
            lo, ln = out[:3].astype(np.int64), out[3:].astype(np.int64)
            assert ln[0] > 0
            assert ((lo + ln <= UNDEF) | (ln == 0)).all()
