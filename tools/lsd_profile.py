"""Time the LSD rectangle validation kernels (k_lsd_validate, k_lsd_improve) alone on the benchmark's LSD call.

    python tools/lsd_profile.py [--reps 4] [--root DIR[,DIR...]] [--rounds 1] [--out DIR]

The call is the one bench.py makes: 3168 frames cycling through the 256 frames of synth.render_sequence_parallel(seed=2, n=256), LSD_REFINE_ADV.
Every kernel of the call is timed with the library's event-bracketed launch profile (the source of bench.py's roofline.per_kernel); the context set-up
(lsd_alloc: buffers and tables) is timed with a host clock around a synchronising call.  --root imports planarslam_b200 from one or more trees, each in
its own child process, alternating over --rounds, so that two builds can be compared in one command.  One JSON line per child; with --out, the segments
of the last call (end points, width, precision, log-NFA for every frame) are written to DIR/lsd_<tag>.npz for a byte comparison between trees.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_FRAMES, DISTINCT = 3168, 256


def _child(args):
    sys.path.insert(0, args.root)
    import numpy as np
    from planarslam_b200._lib import Context

    gray = np.load(args.frames)["gray"]
    frames = np.ascontiguousarray(gray[np.arange(N_FRAMES) % DISTINCT])
    ctx = Context(640, 480, N_FRAMES)
    L = ctx.L
    t0 = time.perf_counter()
    ctx.check(L.pslam_lsd_set_rect_enumeration(ctx.h, 1))              # allocates the LSD context (synchronises)
    setup_ms = (time.perf_counter() - t0) * 1e3
    cap = int(L.pslam_lsd_max_segments(ctx.h))
    segs, wpn, cnt = np.zeros((N_FRAMES, cap, 4), np.float32), np.zeros((N_FRAMES, cap, 3)), np.zeros(N_FRAMES, np.int32)

    def call():
        ctx.check(L.pslam_lsd_detect_batch(ctx.h, frames.ctypes.data, N_FRAMES, 2, segs.ctypes.data, wpn.ctypes.data, cap, cnt.ctypes.data))

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
    res = {"tag": args.tag, "root": args.root, "frames": N_FRAMES, "reps": args.reps, "context_setup_ms": round(setup_ms, 1),
           "segments_per_frame": float(cnt.mean()), "ms_per_call": per,
           "validate_plus_improve_ms": round(per.get("lsd_validate", 0) + per.get("lsd_improve", 0), 3)}
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        m = np.arange(cap)[None, :] < cnt[:, None]
        np.savez(os.path.join(args.out, f"lsd_{args.tag}.npz"), n=cnt, segs=segs[m], width=wpn[m][:, 0], prec=wpn[m][:, 1], nfa=wpn[m][:, 2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--root", default=ROOT, help="comma-separated trees to time")
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--out", default=None)
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
    gray, _ = synth.render_sequence_parallel(seed=2, n=DISTINCT, workers=max(1, min(64, cores)))
    with tempfile.TemporaryDirectory() as tmp:
        fpath = os.path.join(tmp, "frames.npz")
        np.savez(fpath, gray=gray)
        roots = [os.path.abspath(r) for r in args.root.split(",")]
        for rnd in range(args.rounds):
            for i, root in enumerate(roots):
                tag = f"t{i}_r{rnd}"
                cmd = [sys.executable, os.path.abspath(__file__), "--child", "--reps", str(args.reps), "--root", root, "--frames", fpath,
                       "--tag", tag] + (["--out", args.out] if args.out and rnd == 0 else [])
                subprocess.run(cmd, check=True)


if __name__ == "__main__":
    main()
