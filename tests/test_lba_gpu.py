"""GPU: Optimizer::LocalBundleAdjustment through the C ABI vs the CPU oracle (BASELINE.json config 4 shape).

Bar (BASELINE.json north_star): SE3 pose within 1e-4 rad / 1e-3 m of the reference path after the same LM iteration
count.  The two implementations share the summation order of H_ll, H_pp, b and of the Schur terms; they differ in libm
ulps (sin / cos / atan2 inside the plane edges' numeric Jacobians, se3 exp) and in the tree-shaped chi2 reductions, so the
tolerances used here are far tighter than the bar: 1e-6 rad / 1e-6 m on key-frame poses,
1e-4 m on landmarks (two-view points at 4 m depth amplify the pose difference to ~1e-5 m), identical erase
lists and identical LM iteration / trial counts.  A points-only problem (no libm on the path beyond se3 exp's small-angle
branch) must agree bit for bit."""
import numpy as np
import pytest

import oracle_lib
from planarslam_b200 import synth_lba, synth_pose

pytestmark = pytest.mark.gpu
ROT_TOL, TRANS_TOL, LM_TOL = 1e-6, 1e-6, 1e-4


def _compare(r, o, tag=""):
    for k in range(len(r["kf_Tcw_d"])):
        er, et = synth_pose.pose_error(r["kf_Tcw_d"][k], o["kf_Tcw_d"][k])
        assert er < ROT_TOL and et < TRANS_TOL, (tag, k, er, et, r["iterations"], o["iterations"], r["trials"], o["trials"], r["chi2"], o["chi2"])
    assert np.abs(r["kf_Tcw"] - o["kf_Tcw"]).max() < 1e-5
    assert np.abs(r["pt_Xw_d"] - o["pt_Xw_d"]).max() < LM_TOL if r["pt_Xw_d"].size else True
    assert np.abs(r["line_Xw_d"] - o["line_Xw_d"]).max() < LM_TOL if r["line_Xw_d"].size else True
    assert np.abs(r["plane_Xw_d"] - o["plane_Xw_d"]).max() < LM_TOL if r["plane_Xw_d"].size else True
    assert np.abs(r["pt_Xw"] - o["pt_Xw"]).max() < 2 * LM_TOL if r["pt_Xw"].size else True
    assert r["iterations"] == o["iterations"], (tag, r["iterations"], o["iterations"])
    assert r["trials"] == o["trials"], (tag, r["trials"], o["trials"])
    assert np.allclose(r["chi2"], o["chi2"], rtol=1e-5), (tag, r["chi2"], o["chi2"])
    assert np.array_equal(r["erase_pt"], o["erase_pt"]), tag
    assert np.array_equal(r["erase_line"], o["erase_line"]), tag
    for t in range(3):
        assert np.array_equal(r["erase_plane"][t], o["erase_plane"][t]), (tag, t)


def test_lba_config4_matches_oracle():
    from planarslam_b200.lba import LocalBundleAdjuster
    ba = LocalBundleAdjuster()
    probs = [synth_lba.make_lba_problem(s) for s in range(3)]                 # 20 KFs, 5000 point + 200 line + 30 plane edges
    res = ba.LocalBundleAdjustmentBatch(probs)
    for i, (p, r) in enumerate(zip(probs, res)):
        o = oracle_lib.local_bundle_adjustment(p)
        _compare(r, o, tag=f"problem {i}")
        e0 = np.mean([synth_pose.pose_error(p["kf_Tcw"][k], p["kf_Tcw_true"][k]) for k in range(1, 20)], 0)
        e1 = np.mean([synth_pose.pose_error(r["kf_Tcw_d"][k], p["kf_Tcw_true"][k]) for k in range(1, 20)], 0)
        assert e1[0] < e0[0] and e1[1] < e0[1]                                # and it moves towards the ground truth


def test_lba_edge_mixes_and_single_call():
    from planarslam_b200.lba import LocalBundleAdjuster
    ba = LocalBundleAdjuster()
    cases = [dict(n_kf=8, n_fixed=2, n_points=400, n_pt_obs=2400, n_lines=20, n_line_obs=40, n_plane_obs=(8, 2, 2)),
             dict(n_kf=6, n_fixed=1, n_points=300, n_pt_obs=1500, n_lines=0, n_line_obs=0, n_plane_obs=(0, 0, 0), outlier_frac=0.0, mono_frac=0.0),
             dict(n_kf=12, n_fixed=2, n_points=300, n_pt_obs=2400, n_lines=4, n_line_obs=40, n_plane_obs=(12, 4, 4), line_norm3=False, outlier_frac=0.2,
                  kf_stride=5, plane_outlier_frac=0.25),                                # line / plane gates fire, rejected LM trials
             dict(n_kf=5, n_fixed=1, n_points=200, n_pt_obs=900, n_lines=30, n_line_obs=60, n_plane_obs=(6, 2, 1), line_kf_quirk=True),
             dict(n_kf=3, n_fixed=1, n_points=50, n_pt_obs=140, n_lines=0, n_line_obs=0, n_plane_obs=(0, 0, 0)),
             dict(n_kf=40, n_fixed=4, n_points=1200, n_pt_obs=6000, n_lines=40, n_line_obs=80, n_plane_obs=(20, 4, 4), kf_stride=1)]   # S in global memory
    for i, kw in enumerate(cases):
        p = synth_lba.make_lba_problem(50 + i, **kw)
        r = ba.LocalBundleAdjustment(p)
        o = oracle_lib.local_bundle_adjustment(p)
        _compare(r, o, tag=f"case {i}")


def test_lba_points_only_is_bit_exact():
    from planarslam_b200.lba import LocalBundleAdjuster
    ba = LocalBundleAdjuster()
    p = synth_lba.make_lba_problem(5, n_kf=6, n_fixed=1, n_points=300, n_pt_obs=1500, n_lines=0, n_line_obs=0, n_plane_obs=(0, 0, 0),
                                   outlier_frac=0.0, mono_frac=0.0)
    r, o = ba.LocalBundleAdjustment(p), oracle_lib.local_bundle_adjustment(p)
    assert np.array_equal(r["kf_Tcw_d"], o["kf_Tcw_d"]) and np.array_equal(r["pt_Xw_d"], o["pt_Xw_d"])
    assert np.array_equal(r["kf_Tcw"], o["kf_Tcw"]) and np.array_equal(r["pt_Xw"], o["pt_Xw"])
    assert r["iterations"] == o["iterations"] and r["trials"] == o["trials"]


def test_lba_invalid_inputs():
    from planarslam_b200.lba import LocalBundleAdjuster
    from planarslam_b200._lib import PslamError
    ba = LocalBundleAdjuster()
    p = synth_lba.make_lba_problem(1, n_kf=3, n_fixed=1, n_points=20, n_pt_obs=50, n_lines=0, n_line_obs=0, n_plane_obs=(0, 0, 0))
    p["pt_obs_kf"] = p["pt_obs_kf"].copy()
    p["pt_obs_kf"][0] = 99
    with pytest.raises(PslamError):
        ba.LocalBundleAdjustment(p)
