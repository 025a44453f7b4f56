"""Cost of the map plane updates in the planar tracking chain (pslam_track_planar_set_map_plane_updates).

    python tools/track_planar_mapplanes_profile.py [--frames 256] [--rounds 3] [--out DIR]

Sequence and map as tools/track_planar_profile.py: frames 0 .. N-1 of the synthetic room corner, resident in HBM, against the snapshot of
synth_planar_map.build_planar_map (every 32nd frame a key frame).  Run 1: whole pslam_track_planar_sequence_dev calls timed with CUDA events on the context's
stream, alternating updates off / on --rounds times (the snapshot is re-uploaded before every call, outside the timed region, so every call with updates
starts from the same clouds).  Run 2, separate: one call with updates on and pslam_profile_enable, for k_planar_map_plane_update's per-launch time.  Prints the
card's name and power limit and one JSON line; --out also writes it to DIR/track_planar_mapplanes.json.
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
    from planarslam_b200.tracking import PLANAR_STATS, PlanarTracker

    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    n = a.frames
    ctx = Context(640, 480, max_batch=n)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    frames = [synth.render_frame(2, f, n_frames=n)[:2] for f in range(n)]
    m = build_planar_map(ctx, list(range(0, n, 32)), n_frames=n)
    tr = PlanarTracker(ctx)
    with torch.cuda.stream(stream):
        g = torch.from_numpy(np.stack([f[0] for f in frames])).cuda()
        d = torch.from_numpy(np.stack([f[1] for f in frames]).view(np.int16)).cuda()
    stream.synchronize()
    L = ctx.L
    L.pslam_track_planar_sequence_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p] + [C.c_void_p] * 6
    T0 = np.ascontiguousarray(synth_map.true_pose(0, n), np.float32)
    R0 = (T0[:3, :3].astype(np.float64) @ m["R_cm"].astype(np.float64)).astype(np.float32)
    poses, Rcm, st = np.zeros((n, 4, 4), np.float32), np.zeros((n, 3, 3), np.float32), np.zeros((n, PLANAR_STATS), np.int32)

    def run():
        ctx.check(L.pslam_track_planar_sequence_dev(ctx.h, g.data_ptr(), d.data_ptr(), n, C.byref(tr.params), T0.ctypes.data, None, R0.ctypes.data,
                                                    poses.ctypes.data, Rcm.ctypes.data, st.ctypes.data))

    def timed(on):
        tr.update_map_planes = on
        tr.set_map(m)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        run()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1)

    timed(False); timed(True)
    ms = {"updates_off": [], "updates_on": []}
    for _ in range(a.rounds):
        ms["updates_off"].append(timed(False))
        ms["updates_on"].append(timed(True))
    res = {"card": card, "frames": n, "rounds": a.rounds}
    for k, v in ms.items():
        res[k] = {"ms_per_sequence": [round(x, 2) for x in v], "ms_per_frame_best": round(min(v) / n, 4), "frames_per_sec_best": round(n * 1000.0 / min(v), 1)}
    off, pts = tr.map_planes()
    res["map_plane_points_after"] = [int(x) for x in np.diff(off)]
    res["map_plane_points_upload"] = [int(x) for x in np.diff(m["planes"]["pts_off"])]
    rows = tr.plane_matches(n)
    res["merges_per_frame"] = round(float((rows[:, 0] >= 0).sum()) / n, 2)
    # run 2: the update kernel alone, with the per-launch profiler on
    tr.update_map_planes = True
    tr.set_map(m)
    ctx.profile(True)
    run()
    rep = ctx.profile_report()
    ctx.profile(False)
    launches, total = rep.get("planar_map_plane_update", (0, 0.0))
    res["planar_map_plane_update"] = {"launches": launches, "total_ms": round(total, 3), "us_per_launch": round(1000.0 * total / max(launches, 1), 2)}
    print("card:", card)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "track_planar_mapplanes.json"), "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
