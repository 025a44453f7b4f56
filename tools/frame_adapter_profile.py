"""What pslam_adapter::ref::FrameConstructor::batch() adds to the RGB-D Frame constructor call: the host time per frame of unpacking the call's outputs into
the reference's Frame objects (cv::KeyPoint / KeyLine / cv::Mat / PCL clouds / SurfaceNormal / the 64x48 grid / FrameLine with compPt3dCov per supporting
sample), next to the time of pslam_frame_construct_batch alone on the same 640x480 batches (page-locked buffers in both).

The adapter fills the reference's own Frame class, so this needs the test library oracle/_ref/libframe_adapter_ref.so (built from the reference tree by
__graft_entry__.build()).  Prints one JSON line with the card name and power limit read in the same run; --out also writes it to
DIR/frame_adapter_profile.json."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _card():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock"], info["sm_clock_max"] = [v.strip() for v in q.split(",")]
    except Exception as e:     # the numbers are still printed, without the card's settings
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU and has no CPU mode")
    import test_frame_adapter_gpu as T
    from depth_cameras import frames
    from planarslam_b200.frame import ConstructFrames, FrameOutputs
    if not os.path.exists(T.LIB):
        raise SystemExit(f"{T.LIB} not built (it needs the reference tree at build time)")
    B = args.batch
    gray, depth = frames("tum3", B, seed=3)
    L = T.lib()

    # pslam_frame_construct_batch alone, page-locked outputs
    ctx = T.Context(640, 480, B, fx=T.CASES["tum3"][2][0], fy=T.CASES["tum3"][2][1], cx=T.CASES["tum3"][2][2], cy=T.CASES["tum3"][2][3],
                    depth_scale=T.scale_of(5000.0))
    out = FrameOutputs(ctx, B, cap_plane_pts=T.CAP_PTS, pinned=True)
    g_p = torch.from_numpy(gray).pin_memory().numpy()
    d_p = torch.from_numpy(depth).pin_memory().numpy()
    for _ in range(3):
        ConstructFrames(ctx, g_p, d_p, out, bf=T.BF, plane_dist_th=T.PLANE_TH)
    t0 = time.perf_counter()
    for _ in range(args.calls):
        ConstructFrames(ctx, g_p, d_p, out, bf=T.BF, plane_dist_th=T.PLANE_TH)      # returns after its stream synchronise
    construct_s = (time.perf_counter() - t0) / (args.calls * B)

    # batch(): the same call through the adapter, then the unpacking into Frames
    A = T.Adapter("tum3", max_batch=B)
    stamps = np.arange(B, dtype=np.float64)
    for f in A.batch(gray, depth, stamps):
        L.fad_free_frame(f)
    t_warm = np.zeros(3)
    L.fad_timing(A.hnd, t_warm.ctypes.data)
    t0 = time.perf_counter()
    for _ in range(args.calls):
        for f in A.batch(gray, depth, stamps):
            L.fad_free_frame(f)
    batch_s = (time.perf_counter() - t0) / (args.calls * B)
    t_end = np.zeros(3)
    L.fad_timing(A.hnd, t_end.ctypes.data)
    call_s, unpack_s, support_s = (t_end - t_warm) / (args.calls * B)
    A.close()
    res = {"card": _card(), "frames_per_call": B, "calls": args.calls, "size": "640x480",
           "construct_batch_ms_per_frame": round(construct_s * 1e3, 4),
           "adapter_call_ms_per_frame": round(call_s * 1e3, 4),
           "adapter_unpack_ms_per_frame": round(unpack_s * 1e3, 4),
           "of_which_frameline_support_ms_per_frame": round(support_s * 1e3, 4),
           "adapter_batch_ms_per_frame": round(batch_s * 1e3, 4),
           "unpack_over_construct": round(unpack_s / construct_s, 4)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "frame_adapter_profile.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
