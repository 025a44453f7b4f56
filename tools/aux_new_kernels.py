"""Auxiliary GPU leg for bench.py: throughput + result signatures of the two kernels added after the round-1 GPU budget was spent
(k_lines3d = Frame::isLineGood, k_track_manhattan = Tracking::TrackManhattanFrame).  Runs in its OWN process so that a fault in an
as yet GPU-unvalidated kernel cannot touch the headline measurement.  No torch, no oracle: the expected signatures were computed on
the CPU at commit time (tools/make_aux_expected.py -> tests/golden/aux_new_kernels_expected.json) and are only compared here.
Prints one JSON object."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_BASE = 8
BATCH = 1056           # 8 frames per SM of an H100 SXM (132 SMs)


def lines3d_signature(out, drawn):
    v = out["valid"].astype(bool)
    return {"n_valid": int(v.sum()), "n_inliers": int(out["n_inliers"].sum()), "n_points": int(out["n_points"].sum()), "n_drawn": int(drawn.sum()),
            "ab_sum": float(np.round(out["A"][v].sum() + out["B"][v].sum(), 6))}


def manhattan_signature(res):
    return {"found": [int(x) for x in res["found"].ravel()], "n_cone": [int(x) for x in res["n_cone"].ravel()],
            "n_selected": [int(x) for x in res["n_selected"].ravel()], "R_1e4": [int(x) for x in np.rint(res["R"].ravel().astype(np.float64) * 1e4)]}


def main():
    from planarslam_b200 import synth
    from planarslam_b200._lib import Context
    from planarslam_b200.lines import KEYLINE_DTYPE, LineSegment, isLineGood
    from planarslam_b200.manhattan import TrackManhattanFrame
    from planarslam_b200.synth_manhattan import make_manhattan
    out = {}
    exp_path = os.path.join(ROOT, "tests", "golden", "aux_new_kernels_expected.json")
    expected = json.load(open(exp_path)) if os.path.exists(exp_path) else {}
    frames = [synth.render_frame(seed=s, frame=3 * s) for s in range(N_BASE)]
    gray = np.stack([f[0] for f in frames])
    d16 = np.stack([f[1] for f in frames])
    ctx = Context(640, 480, max_batch=N_BASE)
    ls = LineSegment(ctx)
    ext = ls.ExtractLineSegment(gray, 40)
    kl = np.zeros((N_BASE, 40), KEYLINE_DTYPE)
    nl = np.zeros(N_BASE, np.int32)
    for f in range(N_BASE):
        nl[f] = len(ext[f][0])
        kl[f, :nl[f]] = ext[f][0]
    factor = np.float32(1.0 / synth.DEPTH_FACTOR)
    o, drawn = isLineGood(ctx, kl, nl, d16, synth.TUM3_K, factor, seed=1)
    sig = lines3d_signature(o, drawn)
    out["lines3d"] = {"signature": sig, "matches_cpu_expectation": (sig == expected.get("lines3d")) if "lines3d" in expected else None}
    rep = BATCH // N_BASE
    klb, nlb, db = np.tile(kl, (rep, 1)), np.tile(nl, rep), np.tile(d16, (rep, 1, 1))
    isLineGood(ctx, klb, nlb, db, synth.TUM3_K, factor, seed=1)            # warm-up (allocations)
    t0 = time.perf_counter()
    ob, _ = isLineGood(ctx, klb, nlb, db, synth.TUM3_K, factor, seed=1)
    dt = time.perf_counter() - t0
    out["lines3d"]["frames_per_sec_host_buffers"] = round(BATCH / dt, 1)
    out["lines3d"]["batch_consistent"] = bool(all(np.array_equal(ob[:N_BASE][k], o[k], equal_nan=(k == "director")) for k in o.dtype.names))
    data = [make_manhattan(s) for s in range(N_BASE)]
    res, _, _ = TrackManhattanFrame(ctx, np.stack([d[0] for d in data]), [d[1] for d in data], [d[2] for d in data])
    sig = manhattan_signature(res)
    exp = expected.get("manhattan")
    ok = None
    if exp:
        ok = sig["found"] == exp["found"] and sig["n_cone"] == exp["n_cone"] and sig["n_selected"] == exp["n_selected"] and \
            max(abs(a - b) for a, b in zip(sig["R_1e4"], exp["R_1e4"])) <= 1
    out["manhattan"] = {"signature": {k: sig[k] for k in ("found", "n_cone")}, "matches_cpu_expectation": ok}
    Rb = np.tile(np.stack([d[0] for d in data]), (rep, 1, 1))
    nb, dbm = [d[1] for d in data] * rep, [d[2] for d in data] * rep
    TrackManhattanFrame(ctx, Rb, nb, dbm)
    t0 = time.perf_counter()
    TrackManhattanFrame(ctx, Rb, nb, dbm)
    dt = time.perf_counter() - t0
    out["manhattan"]["frames_per_sec_host_buffers"] = round(BATCH / dt, 1)
    out["note"] = f"host-buffer calls (copies and packing included), {BATCH} frames per call; warp-per-frame kernels (k_lines3d_warp, k_track_manhattan_warp)"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
