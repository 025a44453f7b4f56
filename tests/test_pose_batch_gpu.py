"""GPU: the batched PoseOptimization kernel at the benchmark's batch size and across its layout's size range.

The benchmark packs 1584 problems per call (one resident wave on an H100), cycling through 256 distinct ones; a seeded
sample of them is checked against the CPU oracle with the bar of test_pose_gpu.py, and the repeats must come out
bit-identical to their first occurrence.  Problems with thousands of point edges, translation-only problems and the
determinism of two identical calls are checked as well."""
import numpy as np
import pytest

import oracle_lib
from planarslam_b200 import synth_pose
from test_pose_gpu import _compare

pytestmark = pytest.mark.gpu
N_BATCH, DISTINCT = 1584, 256


def _bench_problems():
    base = [synth_pose.make_pose_problem(11 + k // 64, frame=k % 64) for k in range(DISTINCT)]
    return [base[k % DISTINCT] for k in range(N_BATCH)]


def _compare_converged(r, o, tag):
    """test_pose_gpu._compare with the slack it gives its ill-conditioned case (x100 on pose and chi2) and two LM iterations per
    round instead of one.  On the benchmark's problems a round can stop two iterations apart from the oracle: at convergence
    the sign of a chi2 gain of ~1e-12 relative depends on the summation order, and a step that the oracle accepts can be
    rejected ten times here, which ends the round (DESIGN.md §5.6); the pose then differs at the 1e-6 level (measured
    3.2e-7 rad / 1.2e-6 m), 100x inside the required 1e-4 rad / 1e-3 m.  Flags, inlier counts and per-round outlier counts
    are exact."""
    er, et = synth_pose.pose_error(r["Tcw_d"], o["Tcw_d"])
    assert er < 1e-5 and et < 1e-5, (tag, er, et)
    assert r["n_inliers"] == o["n_inliers"], tag
    for k in ("outlier_pt", "outlier_line", "outlier_plane", "outlier_par", "outlier_ver"):
        assert np.array_equal(r[k], o[k]), (tag, k)
    assert np.array_equal(r["trace_i"][:, 2], o["trace_i"][:, 2]), (tag, r["trace_i"], o["trace_i"])
    assert np.abs(r["trace_i"][:, 0] - o["trace_i"][:, 0]).max() <= 2, (tag, r["trace_i"], o["trace_i"])
    assert np.allclose(r["trace_d"][:, 0], o["trace_d"][:, 0], rtol=1e-4, atol=1e-9), (tag, r["trace_d"], o["trace_d"])


def _same_bytes(a, b):
    for k in ("Tcw", "Tcw_d", "trace_i", "trace_d", "outlier_pt", "outlier_line", "outlier_plane", "outlier_par", "outlier_ver"):
        assert a[k].tobytes() == b[k].tobytes(), k
    assert a["n_inliers"] == b["n_inliers"]


def test_bench_batch_matches_oracle():
    from planarslam_b200.optimizer import Optimizer
    probs = _bench_problems()
    res = Optimizer().PoseOptimizationBatch(probs)
    for k in np.random.default_rng(2024).choice(N_BATCH, 24, replace=False):
        _compare_converged(res[k], oracle_lib.pose_optimization(probs[k]), f"problem {k}")
    for k in range(DISTINCT, N_BATCH):          # repeats of a problem give the same bytes wherever they sit in the batch
        _same_bytes(res[k], res[k % DISTINCT])


def test_large_and_small_problems_in_one_batch():
    from planarslam_b200.optimizer import Optimizer
    probs = [synth_pose.make_pose_problem(300, frame=1, n_points=6000, n_lines=120, n_planes=6, n_par=2, n_ver=3, outlier_frac=0.1),
             synth_pose.make_pose_problem(301, frame=2, n_points=40, n_lines=0, n_planes=1, n_par=0, n_ver=0),
             synth_pose.make_pose_problem(302, frame=3, n_points=4100, n_lines=0, n_planes=0, n_par=0, n_ver=0),
             synth_pose.make_pose_problem(303, frame=4, n_points=1000, n_lines=40, n_planes=3, n_par=1, n_ver=2)]
    res = Optimizer().PoseOptimizationBatch(probs)
    for i, (p, r) in enumerate(zip(probs, res)):
        _compare(r, oracle_lib.pose_optimization(p), p, tag=f"case {i}")


def test_translation_batch_matches_oracle():
    from planarslam_b200.optimizer import Optimizer
    probs = [synth_pose.make_pose_problem(310 + s, frame=2 * s, n_points=n, n_planes=3, rot_pert=0.0, trans_pert=0.05)
             for s, n in enumerate((1000, 5000, 60, 1000))]
    res = Optimizer().TranslationOptimizationBatch(probs)
    for i, (p, r) in enumerate(zip(probs, res)):
        o = oracle_lib.translation_optimization(p)
        _compare(r, o, p, tag=f"case {i}")
        assert np.abs(r["Tcw_d"][:3, :3] - o["Tcw_d"][:3, :3]).max() < 1e-12     # the rotation block is untouched


def test_two_identical_calls_give_identical_bytes():
    from planarslam_b200.optimizer import Optimizer
    opt = Optimizer()
    probs = _bench_problems()[:528] + [synth_pose.make_pose_problem(320, n_points=3000, n_lines=60, n_planes=4, n_par=1, n_ver=1)]
    opt.pack(probs)
    opt.run_packed()
    a = opt.fetch()
    opt.run_packed()
    b = opt.fetch()
    for x, y in zip(a, b):
        _same_bytes(x, y)
