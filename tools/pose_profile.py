"""Time k_pose_optimization alone on the benchmark's pose batch and report where its passes go.

    python tools/pose_profile.py [--reps 8] [--threads 32,64,128] [--root DIR] [--out DIR]

The batch is the one bench.py builds: 1584 problems cycling through the 256 distinct problems
synth_pose.make_pose_problem(11 + k // 64, frame=k % 64) (1000 points, 40 lines = 80 edges, 3 + 1 + 2 plane edges).
Each configuration runs in a child process with PSLAM_POSE_THREADS set to its --threads value: builds that took the batch
block size from that variable read it once per process; builds with a fixed block size ignore it, and then --threads
only repeats the measurement.  Configurations: with and without the plane / parallel / vertical plane edges, at every
--threads value.  The kernel is timed with the library's event-bracketed launch profile (the source of
bench.py's roofline.per_kernel); the LM pass counts come from trace_i.  --root imports planarslam_b200 from another
tree, so that two builds can be timed by the same script.  One JSON line per configuration; with --out, the poses,
inlier counts and traces of every configuration are also written to DIR/pose_<tag>.npz.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_PROBLEMS, DISTINCT = 1584, 256
PLANE_KEYS = ("plane_meas", "plane_map", "par_meas", "par_map", "ver_meas", "ver_map")


def _child(args):
    sys.path.insert(0, args.root)
    import numpy as np
    from planarslam_b200 import synth_pose
    from planarslam_b200.optimizer import Optimizer

    base = [synth_pose.make_pose_problem(11 + k // 64, frame=k % 64) for k in range(DISTINCT)]
    if not args.planes:
        base = [{k: (v[:0] if k in PLANE_KEYS else v) for k, v in p.items()} for p in base]
    probs = [base[k % DISTINCT] for k in range(N_PROBLEMS)]
    opt = Optimizer()
    opt.pack(probs)
    for _ in range(3):
        opt.run_packed()
    opt.ctx.synchronize()
    opt.ctx.profile(True)
    for _ in range(args.reps):
        opt.run_packed()
    opt.ctx.synchronize()
    n, ms = opt.ctx.profile_report()["pose_optimization"]
    opt.ctx.profile(False)
    r = opt.fetch()
    ti = np.stack([q["trace_i"] for q in r])                      # [problem, round, (iterations, trials, nBad)], -1: round not run
    ran = ti[:, :, 0] >= 0
    iters = np.where(ran, ti[:, :, 0], 0).sum(1)
    trials = np.where(ran, ti[:, :, 1], 0).sum(1)
    rounds = ran.sum(1)
    edges = np.array([len(p["Xw"]) + 2 * len(p["line_Xw"]) + sum(len(p[k]) for k in ("plane_meas", "par_meas", "ver_meas")) for p in probs])
    res = {"tag": args.tag, "threads": os.environ.get("PSLAM_POSE_THREADS"), "planes": bool(args.planes), "problems": N_PROBLEMS,
           "edges_per_problem": float(edges.mean()), "launches": n, "ms_per_launch": round(ms / n, 4),
           "lm_iterations_per_problem": float(iters.mean()), "trials_per_problem": float(trials.mean()), "rounds_per_problem": float(rounds.mean()),
           # one chi2 pass per trial; an iteration adds one pass (fused error + normal equations) or two (computeActiveErrors, then buildSystem)
           "passes_fused": float((iters + trials).mean()), "passes_unfused": float((2 * iters + trials).mean())}
    res["us_per_problem_pass_fused"] = round(ms / n * 1e3 / (N_PROBLEMS * res["passes_fused"]), 5)
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        np.savez(os.path.join(args.out, f"pose_{args.tag}.npz"), Tcw_d=np.stack([q["Tcw_d"] for q in r]), n_inliers=np.array([q["n_inliers"] for q in r]),
                 trace_i=ti, trace_d=np.stack([q["trace_d"] for q in r]), outlier_pt=np.concatenate([q["outlier_pt"] for q in r]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--threads", default="64")
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--name", default="pr", help="prefix of the configuration tags")
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--planes", type=int, default=1, help=argparse.SUPPRESS)
    ap.add_argument("--tag", default="", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return _child(args)
    for planes in (1, 0):
        for nt in args.threads.split(","):
            tag = f"{args.name}_t{nt}_{'planes' if planes else 'noplanes'}"
            cmd = [sys.executable, os.path.abspath(__file__), "--child", "--reps", str(args.reps), "--root", os.path.abspath(args.root),
                   "--planes", str(planes), "--tag", tag] + (["--out", args.out] if args.out else [])
            subprocess.run(cmd, check=True, env=dict(os.environ, PSLAM_POSE_THREADS=nt))


if __name__ == "__main__":
    main()
