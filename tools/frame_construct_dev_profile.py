"""Time the Frame constructor on device-resident frames against the same stages chained call by call, and the colour conversion in front of it.

    python tools/frame_construct_dev_profile.py [--frames 1584] [--rounds 3] [--distinct 64] [--out DIR]

One context (640x480, TUM3 camera, max_batch = --frames) runs, alternating over --rounds:
  (a) dev     pslam_frame_construct_batch_dev on grey + depth frames in HBM (construct_frames_dev)
  (b) chain   the same seven stages as separate _dev calls, in the same order, into caller-allocated tensors - PEAC, plane post-processing, surface
              normals, ORB, stereo, lines + LBD, isLineGood - as bench.py's device leg calls them (there each family has its own context and stream)
  (c) color   (a) behind pslam_gray_from_color_batch_dev on RGB frames whose grey is the grey of (a)
Each is timed with CUDA events around one call (the per-frame time is that over --frames).  The conversion kernel alone is timed over 20 back-to-back
launches per channel count; achieved bytes/s = (channels + 1) bytes per pixel over the kernel time, against the 3.35 TB/s of the H100 SXM data sheet.
The frames cycle through --distinct renders of synth.render_sequence_parallel(seed=2).  (a) and (b) must return the same products: the tool checks the
counts and the key points of every frame.  Prints one JSON line with the card name, its power limit and SM clocks; --out also writes it to
DIR/frame_construct_dev_profile.json.
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
HBM_PEAK = 3.35e12


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
    ap.add_argument("--frames", type=int, default=1584)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--distinct", type=int, default=64)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    from planarslam_b200 import synth
    from planarslam_b200._lib import PLANE_DTYPE, Context
    from planarslam_b200.frame import CUDA_STREAM_LEGACY, FrameOutputs, construct_frames_dev, gray_from_color
    from planarslam_b200.lines import KEYLINE_DTYPE, LINE3D_DTYPE
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU and has no CPU mode")
    N, W, H = args.frames, 640, 480
    g0, d0 = synth.render_sequence_parallel(2, args.distinct)
    idx = np.arange(N) % args.distinct
    dev = torch.device("cuda:0")
    gray = torch.from_numpy(g0[idx]).to(dev)
    depth = torch.from_numpy(d0[idx].view(np.int16)).to(dev)
    # R = G = B = grey: the weights sum to 2^15, so the conversion returns the grey frames and (c) does the work of (a) plus the conversion
    rgb = torch.stack([gray, gray, gray], -1).contiguous()
    rgba = torch.cat([rgb, torch.full_like(gray, 255)[..., None]], -1).contiguous()
    ctx = Context(W, H, N)
    L = ctx.L
    cap, maxp, n_sn = int(L.pslam_orb_max_keypoints(ctx.h)), int(L.pslam_peac_max_planes(ctx.h)), int(L.pslam_surface_normals_count(ctx.h))
    MAX_LINES, PP_CAP, BF, DIST_TH = 40, 4096, 40.0, 0.05
    df = float(ctx.cfg.depth_scale)
    kw = dict(bf=BF, plane_dist_th=DIST_TH, line_seed=1, max_lines=MAX_LINES, cap_plane_pts=PP_CAP, normals=True)
    out_a = FrameOutputs(ctx, N, MAX_LINES, PP_CAP, True, device=dev)
    out_c = FrameOutputs(ctx, N, MAX_LINES, PP_CAP, True, device=dev)
    # (b): the caller's buffers for the chained calls
    e = lambda shape, dt: torch.empty(shape, dtype=dt, device=dev)   # noqa: E731
    labels, members = e((N, H * W), torch.int32), e((N, H * W), torch.int32)
    planes, npl, moff = e((N, maxp, PLANE_DTYPE.itemsize), torch.uint8), e(N, torch.int32), e((N, maxp + 1), torch.int32)
    pp_n, pp_src, pp_coef, pp_off = e(N, torch.int32), e((N, maxp), torch.int32), e((N, maxp, 4), torch.float32), e((N, maxp + 1), torch.int32)
    pp_pts, pp_st, sn8 = e((N, PP_CAP, 3), torch.float32), e(N, torch.int32), e((N, n_sn, 8), torch.float32)
    kps, desc, nk, ur, dz = e((N, cap, 28), torch.uint8), e((N, cap, 32), torch.uint8), e(N, torch.int32), e((N, cap), torch.float32), e((N, cap), torch.float32)
    kl, lf, ld = e((N, MAX_LINES, KEYLINE_DTYPE.itemsize), torch.uint8), e((N, MAX_LINES, 3), torch.float64), e((N, MAX_LINES, 32), torch.uint8)
    l3d, nkl, drawn = e((N, MAX_LINES, LINE3D_DTYPE.itemsize), torch.uint8), e(N, torch.int32), e(N, torch.int32)
    seed = torch.ones(N, dtype=torch.int32, device=dev)
    cam4 = (C.c_float * 4)(ctx.cfg.fx, ctx.cfg.fy, ctx.cfg.cx, ctx.cfg.cy)
    P = lambda t: t.data_ptr()   # noqa: E731
    L.pslam_planes_post_batch_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 4 + [C.c_float] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
    L.pslam_surface_normals_batch_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.pslam_lines_extract_describe_batch_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 4

    def chain():
        ctx.check(L.pslam_peac_run_batch_dev(ctx.h, P(depth), N, P(labels), P(planes), P(npl), P(members), P(moff)))
        ctx.check(L.pslam_planes_post_batch_dev(ctx.h, P(depth), N, P(planes), P(npl), P(members), P(moff), DIST_TH, P(pp_n), P(pp_src), P(pp_coef), P(pp_off),
                                                P(pp_pts), PP_CAP, P(pp_st)))
        ctx.check(L.pslam_surface_normals_batch_dev(ctx.h, P(depth), N, P(sn8), None))
        ctx.check(L.pslam_orb_extract_batch_dev(ctx.h, P(gray), N, P(kps), P(desc), cap, P(nk)))
        ctx.check(L.pslam_compute_stereo_from_rgbd_batch_dev(ctx.h, P(kps), P(kps), P(nk), cap, P(depth), N, df, BF, P(ur), P(dz)))
        ctx.check(L.pslam_lines_extract_describe_batch_dev(ctx.h, P(gray), N, MAX_LINES, P(kl), P(lf), P(ld), P(nkl)))
        ctx.check(L.pslam_lines3d_batch_dev(ctx.h, P(kl), P(nkl), MAX_LINES, P(depth), N, df, cam4, P(seed), None, P(l3d), P(drawn)))

    variants = {"dev": lambda: construct_frames_dev(ctx, gray, depth, out=out_a, **kw),
                "chain": chain,
                "color": lambda: construct_frames_dev(ctx, rgb, depth, out=out_c, **kw)}
    st = torch.cuda.current_stream()
    ctx.set_stream(st.cuda_stream or CUDA_STREAM_LEGACY)      # the chained calls run where the events are recorded
    for f in variants.values():        # warm-up: stage buffers, scratch, tensor maps
        f()
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k, f in variants.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
            f()
            b.record(st)
            b.synchronize()
            times[k].append(a.elapsed_time(b))
    # (a) and (b) wrote the same products
    assert torch.equal(out_a.n_keys, nk) and torch.equal(out_a.n_lines, nkl) and torch.equal(out_a.n_planes, pp_n) and not out_a.status.any().item()
    ka, kb = out_a.keys.cpu().numpy(), kps.cpu().numpy()
    nkh = nk.cpu().numpy()
    assert all(ka[f, :nkh[f]].tobytes() == kb[f, :nkh[f]].tobytes() for f in range(N))
    assert torch.equal(gray_from_color(ctx, rgb), gray) and torch.equal(out_c.n_keys, nk)
    # the conversion kernel alone
    conv = {}
    for name, img in (("rgb", rgb), ("rgba", rgba)):
        gray_from_color(ctx, img)
        reps = 20
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        for _ in range(reps):
            gray_from_color(ctx, img)
        b.record(st)
        b.synchronize()
        ms = a.elapsed_time(b) / reps
        nbytes = N * H * W * (img.shape[-1] + 1)
        conv[name] = {"ms_per_launch": round(ms, 4), "us_per_frame": round(1e3 * ms / N, 4), "bytes_per_launch": nbytes,
                      "achieved_TBps": round(nbytes / (ms * 1e-3) / 1e12, 3), "share_of_3.35TBps": round(nbytes / (ms * 1e-3) / HBM_PEAK, 3)}
    res = {"card": _card(), "frames": N, "size": [W, H], "rounds": args.rounds,
           "ms_per_call": {k: [round(v, 2) for v in t] for k, t in times.items()},
           "us_per_frame_median": {k: round(1e3 * float(np.median(t)) / N, 2) for k, t in times.items()},
           "gray_from_color": conv}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "frame_construct_dev_profile.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
