"""Latency per frame of the two device-resident tracking chains on the same sequence.

    python tools/track_planar_profile.py [--frames 256] [--rounds 3] [--out DIR]

Sequence: frames 0 .. N-1 of the synthetic room corner (synth.render_frame(2, f, n_frames=N)), 640x480, resident in HBM.  Chains:
  planar  pslam_track_planar_sequence_dev  (Manhattan rotation, TranslationWithMotionModel, TrackLocalMap with point / line / plane edges) against the
          snapshot of synth_planar_map.build_planar_map (every 32nd frame a key frame)
  points  pslam_track_sequence_dev         (TrackWithMotionModel + points-only TrackLocalMap) against the map points of the same snapshot
Each call covers the whole sequence (stage A batched, stage B frame after frame); both are warmed up once, then timed with CUDA events on the context's
stream, alternating planar / points --rounds times.  Prints the card's name and power limit and one JSON line; --out also writes it to DIR/track_planar.json.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    from planarslam_b200 import synth, synth_map
    from planarslam_b200._lib import Context
    from planarslam_b200.synth_planar_map import build_planar_map
    from planarslam_b200.tracking import PLANAR_STATS, PlanarTracker, Tracker

    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    n = a.frames
    ctx = Context(640, 480, max_batch=n)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    frames = [synth.render_frame(2, f, n_frames=n)[:2] for f in range(n)]
    m = build_planar_map(ctx, list(range(0, n, 32)), n_frames=n)
    pts = dict(m["points"]); pts["n"] = len(pts["skip"])
    planar, points = PlanarTracker(ctx), Tracker(ctx)
    planar.set_map(m); points.set_map(pts)
    with torch.cuda.stream(stream):
        g = torch.from_numpy(np.stack([f[0] for f in frames])).cuda()
        d = torch.from_numpy(np.stack([f[1] for f in frames]).view(np.int16)).cuda()
    stream.synchronize()
    L = ctx.L
    L.pslam_track_planar_sequence_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p] + [C.c_void_p] * 6
    L.pslam_track_sequence_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    T0 = np.ascontiguousarray(synth_map.true_pose(0, n), np.float32)
    R0 = (T0[:3, :3].astype(np.float64) @ m["R_cm"].astype(np.float64)).astype(np.float32)
    poses, Rcm, st_p, st_q = (np.zeros((n, 4, 4), np.float32), np.zeros((n, 3, 3), np.float32), np.zeros((n, PLANAR_STATS), np.int32),
                              np.zeros((n, 4), np.int32))

    def run_planar():
        ctx.check(L.pslam_track_planar_sequence_dev(ctx.h, g.data_ptr(), d.data_ptr(), n, C.byref(planar.params), T0.ctypes.data, None, R0.ctypes.data,
                                                    poses.ctypes.data, Rcm.ctypes.data, st_p.ctypes.data))

    def run_points():
        ctx.check(L.pslam_track_sequence_dev(ctx.h, g.data_ptr(), d.data_ptr(), n, C.byref(points.params), T0.ctypes.data, poses.ctypes.data, st_q.ctypes.data))

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1)

    run_planar(); run_points()
    ms = {"planar": [], "points": []}
    for _ in range(a.rounds):
        ms["planar"].append(timed(run_planar))
        ms["points"].append(timed(run_points))
    res = {"card": card, "frames": n, "rounds": a.rounds}
    for k, v in ms.items():
        res[k] = {"ms_per_sequence": [round(x, 2) for x in v], "ms_per_frame_best": round(min(v) / n, 4), "frames_per_sec_best": round(n * 1000.0 / min(v), 1)}
    res["planar_tracked_frames"] = int(st_p[:, 12].sum())
    print("card:", card)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "track_planar.json"), "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
