"""Time the plane post-processing (pslam_planes_post_batch_dev: VoxelGrid, MaxPointDistanceFromPlane, RANSAC refit, compaction) on the benchmark's PEAC call.

    python tools/planes_post_profile.py [--reps 4] [--root DIR[,DIR...]] [--rounds 1] [--out DIR] [--oracle-frames 16]

The call is the one bench.py makes: PEAC on 1584 frames cycling through the 256 frames of synth.render_sequence_parallel(seed=2, n=256), then the
post-processing of its planes.  Every kernel of the call is timed with the library's event-bracketed launch profile (the source of bench.py's
roofline.per_kernel).  --root imports planarslam_b200 from one or more trees, each in its own child process, alternating over --rounds, so that two builds
can be compared in one command.  One JSON line per child, with the shapes the post-processing runs at (planes per frame, members per plane, occupied voxels
of the kept planes); with --out, every output of the last call (n_kept, src, coef, pt_off, the packed points, status) goes to DIR/planes_post_<tag>.npz for a
byte comparison between trees.  The RANSAC iteration counts are not returned by the library; the parent prints their distribution from the CPU oracle
(tests/oracle_lib.planes_post) on --oracle-frames of the frames.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_FRAMES, DISTINCT, DIST_TH, PP_CAP = 1584, 256, 0.05, 4096


def _dist(a):
    import numpy as np
    a = np.asarray(a)
    if a.size == 0:
        return {"n": 0}
    q = np.percentile(a, [50, 90, 99])
    return {"n": int(a.size), "mean": round(float(a.mean()), 1), "p50": float(q[0]), "p90": float(q[1]), "p99": float(q[2]), "max": int(a.max())}


def _child(args):
    sys.path.insert(0, args.root)
    import numpy as np
    import torch
    from planarslam_b200._lib import PLANE_DTYPE, Context

    depth = np.load(args.frames)["depth"]
    H, W = depth.shape[1:]
    dev = torch.device("cuda", 0)
    ctx = Context(W, H, N_FRAMES)
    L = ctx.L
    L.pslam_planes_post_batch_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 4 + [C.c_float] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
    maxp = int(L.pslam_peac_max_planes(ctx.h))
    d_depth = torch.from_numpy(np.ascontiguousarray(depth[np.arange(N_FRAMES) % DISTINCT]).view(np.int16)).to(dev)
    d_labels = torch.empty((N_FRAMES, H * W), dtype=torch.int32, device=dev)
    d_planes = torch.empty((N_FRAMES, maxp, PLANE_DTYPE.itemsize), dtype=torch.uint8, device=dev)
    d_npl = torch.zeros(N_FRAMES, dtype=torch.int32, device=dev)
    d_members = torch.empty((N_FRAMES, H * W), dtype=torch.int32, device=dev)
    d_moff = torch.empty((N_FRAMES, maxp + 1), dtype=torch.int32, device=dev)
    d_n = torch.zeros(N_FRAMES, dtype=torch.int32, device=dev)
    d_src = torch.zeros((N_FRAMES, maxp), dtype=torch.int32, device=dev)
    d_coef = torch.zeros((N_FRAMES, maxp, 4), dtype=torch.float32, device=dev)
    d_off = torch.zeros((N_FRAMES, maxp + 1), dtype=torch.int32, device=dev)
    d_pts = torch.zeros((N_FRAMES, PP_CAP, 3), dtype=torch.float32, device=dev)
    d_status = torch.zeros(N_FRAMES, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    ctx.check(L.pslam_peac_run_batch_dev(ctx.h, d_depth.data_ptr(), N_FRAMES, d_labels.data_ptr(), d_planes.data_ptr(), d_npl.data_ptr(),
                                         d_members.data_ptr(), d_moff.data_ptr()))

    def call():
        ctx.check(L.pslam_planes_post_batch_dev(ctx.h, d_depth.data_ptr(), N_FRAMES, d_planes.data_ptr(), d_npl.data_ptr(), d_members.data_ptr(), d_moff.data_ptr(),
                                                DIST_TH, d_n.data_ptr(), d_src.data_ptr(), d_coef.data_ptr(), d_off.data_ptr(), d_pts.data_ptr(), PP_CAP,
                                                d_status.data_ptr()))

    for _ in range(2):
        call()
    ctx.synchronize()
    ctx.profile(True)
    for _ in range(args.reps):
        call()
    ctx.synchronize()
    rep = ctx.profile_report()
    ctx.profile(False)
    per = {k: round(ms / n, 3) for k, (n, ms) in rep.items()}
    npl, moff = d_npl.cpu().numpy(), d_moff.cpu().numpy()
    n, off, status = d_n.cpu().numpy(), d_off.cpu().numpy(), d_status.cpu().numpy()
    members = np.concatenate([np.diff(moff[f, :min(int(npl[f]), maxp) + 1]) for f in range(N_FRAMES)])
    voxels = np.concatenate([np.diff(off[f, :n[f] + 1]) for f in range(N_FRAMES)])
    res = {"tag": args.tag, "root": args.root, "frames": N_FRAMES, "reps": args.reps, "ms_per_call": per,
           "planes_post_total_ms": round(sum(v for k, v in per.items() if k.startswith("planes_")), 3),
           "planes_per_frame": _dist(npl), "members_per_plane": _dist(members), "voxels_per_kept_plane": _dist(voxels),
           "kept_per_frame": _dist(n), "frames_with_status": int((status != 0).sum())}
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        pts, src, coef = d_pts.cpu().numpy(), d_src.cpu().numpy(), d_coef.cpu().numpy()
        m = np.arange(maxp)[None, :] < n[:, None]
        packed = np.concatenate([pts[f, :off[f, n[f]]] for f in range(N_FRAMES)])
        np.savez(os.path.join(args.out, f"planes_post_{args.tag}.npz"), n_kept=n, src=src[m], coef=coef[m], pt_off=off, pts=packed, status=status)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--root", default=ROOT, help="comma-separated trees to time")
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--out", default=None)
    ap.add_argument("--oracle-frames", type=int, default=16, help="frames whose RANSAC iteration counts the CPU oracle reports (0: none)")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--frames", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--tag", default="", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return _child(args)
    import tempfile

    import numpy as np
    sys.path.insert(0, ROOT)
    from planarslam_b200 import synth
    cores = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    _, depth = synth.render_sequence_parallel(seed=2, n=DISTINCT, workers=max(1, min(64, cores)))
    if args.oracle_frames > 0:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import oracle_lib
        idx = np.linspace(0, DISTINCT - 1, args.oracle_frames).astype(int)
        its = [p["n_iterations"] for f in idx for p in oracle_lib.planes_post(depth[f], dist_th=DIST_TH)]
        print(json.dumps({"oracle_frames": len(idx), "ransac_iterations_per_kept_plane": _dist(its)}), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        fpath = os.path.join(tmp, "frames.npz")
        np.savez(fpath, depth=depth)
        roots = [os.path.abspath(r) for r in args.root.split(",")]
        for rnd in range(args.rounds):
            for i, root in enumerate(roots):
                tag = f"t{i}_r{rnd}"
                cmd = [sys.executable, os.path.abspath(__file__), "--child", "--reps", str(args.reps), "--root", root, "--frames", fpath,
                       "--tag", tag] + (["--out", args.out] if args.out and rnd == args.rounds - 1 else [])
                subprocess.run(cmd, check=True)


if __name__ == "__main__":
    main()
