"""CPU: planarslam_b200/csrc/manhattan_body.h - the code the CUDA kernel k_track_manhattan runs, one thread per frame - compiled for
the HOST with g++ and compared with the oracle (oracle/manhattan.cc, an independent statement with index lists and the generic
Jacobi SVD).  Counts, found flags and membership masks must be identical, the rotation equal to float rounding.  The kernels
themselves are checked on an H100 by tests/test_manhattan_gpu.py and tests/test_cuda_vs_reference_functions_gpu.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_lib
from planarslam_b200.manhattan import MANHATTAN_RESULT_DTYPE
from planarslam_b200.synth_manhattan import make_manhattan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("manhattan") / "libmanhattan_host.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math",
                    "-I", os.path.join(ROOT, "planarslam_b200", "csrc"), "-o", str(out), os.path.join(ROOT, "tests", "host_harness", "manhattan_host.cc")], check=True)
    L = C.CDLL(str(out))
    L.host_track_manhattan.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def host_track(L, R_last, normals, dirs):
    R = np.ascontiguousarray(R_last, np.float32)
    N = np.ascontiguousarray(normals, np.float32).reshape(-1, 3)
    D = np.ascontiguousarray(dirs, np.float64).reshape(-1, 3)
    res = np.zeros(1, MANHATTAN_RESULT_DTYPE)
    nm, dm = np.zeros(max(len(N), 1), np.uint8), np.zeros(max(len(D), 1), np.uint8)
    L.host_track_manhattan(R.ctypes.data, N.ctypes.data, len(N), D.ctypes.data, len(D), res.ctypes.data, nm.ctypes.data, dm.ctypes.data)
    return res[0], nm[:len(N)], dm[:len(D)]


def compare(p, nm, dm, o, atol=2e-6):
    for k in ("found", "n_cone", "n_selected"):
        assert np.array_equal(p[k], o[k]), k
    assert p["min_num"] == o["min_num"] and p["svd_applied"] == o["svd_applied"]
    assert np.allclose(p["R"], o["R"], rtol=0, atol=atol) and np.allclose(p["density"], o["density"], rtol=1e-6, atol=0)
    assert np.array_equal(nm & 7, o["normal_mask"]) and np.array_equal(dm & 7, o["dir_mask"])
    for a in range(3):
        assert int(((nm >> (4 + a)) & 1).sum()) == o["n_cone"][a]


def test_body_matches_oracle(host_lib):
    cases = [dict(seed=s) for s in range(6)]
    cases += [dict(seed=3, weights=(0.5, 0.5, 0.0), clutter=0.02, n_lines=0), dict(seed=5, weights=(0.0, 0.5, 0.5), clutter=0.02),
              dict(seed=6, weights=(0.5, 0.0, 0.5), clutter=0.02), dict(seed=4, weights=(1.0, 0.0, 0.0), clutter=0.0, n_lines=0),
              dict(seed=7, n_normals=300, n_lines=40, perturb_deg=8.0), dict(seed=8, clutter=0.9)]
    kinds = set()
    for kw in cases:
        R_last, normals, dirs, _ = make_manhattan(**kw)
        o = oracle_lib.track_manhattan_frame(R_last, normals, dirs)
        p, nm, dm = host_track(host_lib, R_last, normals, dirs)
        compare(p, nm, dm, o)
        kinds.add((int(o["found"].sum()), tuple(o["found"])))
    assert {k[0] for k in kinds} >= {1, 2, 3} and len([k for k in kinds if k[0] == 2]) == 3          # all three cross-product branches


def test_body_empty_inputs(host_lib):
    R_last = np.eye(3, dtype=np.float32)
    p, nm, dm = host_track(host_lib, R_last, np.zeros((0, 3), np.float32), np.zeros((0, 3)))
    assert p["found"].sum() == 0 and np.array_equal(p["R"], R_last) and p["svd_applied"] == 0
