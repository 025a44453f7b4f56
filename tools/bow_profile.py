"""Time the batched DBoW2 transform against the resident vocabulary (pslam_bow_set_vocabulary + pslam_bow_transform_batch[_dev]).

Inputs: a full ORBvoc-shaped synthetic vocabulary (k = 10, L = 6, 1,111,111 nodes) and 1584 frames x 1000 ORB-like descriptors (noisy copies of
leaf descriptors), plus real ORB descriptors from pslam_orb_extract_batch_dev on synthetic frames.  Reports the upload time of the vocabulary,
ms per batch call and per frame (CUDA events) with the per-kernel split (pslam_profile_enable, separate run), the per-frame pslam_bow_transform
(which uploads the vocabulary on every call) on a few frames, and, when oracle/_ref/libbow_ref.so is present, the reference's DBoW2 on the host's
cores.  Batch and per-frame timings alternate over rounds.  A sample of frames is checked against the CPU oracle at the timed size.

    python tools/bow_profile.py [--frames 1584] [--rounds 3] [--out results.json]

The last line printed is the JSON result; --out also writes it to a file.
"""
from __future__ import annotations

import argparse
import concurrent.futures as cf
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

KEYS = ("word_id", "word_val", "node_id", "node_off", "node_feat")


def gpu_info():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                        # noqa: BLE001
        return f"unavailable ({e})"


def write_vocabulary_txt_fast(voc, path):
    """ref_lib.write_vocabulary_txt's format without the per-byte str() calls (1.1 M lines)."""
    tab = [str(i).encode() for i in range(256)]
    n = len(voc["word_id"])
    parent = np.zeros(n, np.int64)
    parent[voc["child_id"]] = np.repeat(np.arange(n), np.diff(voc["child_off"]))
    with open(path, "wb") as f:
        f.write(f"{voc['k']} {voc['L']} 0 0".encode())
        for i in range(1, n):
            f.write(b"\n%d %d " % (parent[i], int(voc["word_id"][i] >= 0)) + b" ".join(map(tab.__getitem__, voc["desc"][i].tolist())) +
                    b" " + repr(float(voc["weight"][i])).encode())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1584)
    ap.add_argument("--features", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bow_profile: no CUDA device (this measurement has no CPU fallback)")
    import oracle_lib
    import ref_lib
    from planarslam_b200 import synth, synth_lines as sl
    from planarslam_b200._lib import Context
    from planarslam_b200.matcher import bow_transform
    from planarslam_b200.vocabulary import bow_set_vocabulary

    res = dict(gpu=gpu_info(), frames=a.frames, features=a.features)
    print("GPU:", res["gpu"], flush=True)
    t = time.perf_counter()
    voc = sl.make_vocabulary_full(11, k=10, L=6)
    res["vocabulary_nodes"] = len(voc["word_id"])
    nf, cap = a.frames, a.features
    desc = np.stack([sl.make_features_for_vocabulary(1000 + f, voc, cap) for f in range(nf)])
    n = np.full(nf, cap, np.int32)
    print(f"inputs: {len(voc['word_id'])} nodes, {nf} x {cap} descriptors ({time.perf_counter() - t:.1f} s)", flush=True)

    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)                              # not the legacy default stream: the library and the events share this one
    ctx = Context(640, 480, 1)
    ctx.set_stream(stream.cuda_stream)
    L = ctx.L
    t_set = []
    for _ in range(3):
        t = time.perf_counter()
        bow_set_vocabulary(ctx, voc)
        t_set.append((time.perf_counter() - t) * 1e3)
    res["set_vocabulary_ms"] = t_set
    print(f"pslam_bow_set_vocabulary: {', '.join(f'{x:.1f}' for x in t_set)} ms", flush=True)

    def dev_buffers(d_desc, d_n, frames, cap_):
        o = [torch.empty((frames, cap_), dtype=torch.int32, device=dev), torch.empty((frames, cap_), dtype=torch.float64, device=dev),
             torch.empty((frames, cap_), dtype=torch.int32, device=dev), torch.empty((frames, cap_ + 1), dtype=torch.int32, device=dev),
             torch.empty((frames, cap_), dtype=torch.int32, device=dev), torch.empty((frames, 2), dtype=torch.int32, device=dev)]
        call = lambda: ctx.check(L.pslam_bow_transform_batch_dev(ctx.h, d_desc.data_ptr(), d_n.data_ptr(), cap_, frames, 4, *[x.data_ptr() for x in o]))
        return o, call

    def time_dev(call, iters):
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(iters + 1)]
        ev[0].record(stream)
        for i in range(iters):
            call()
            ev[i + 1].record(stream)
        torch.cuda.synchronize()
        return [ev[i].elapsed_time(ev[i + 1]) for i in range(iters)]

    def kernel_split(call, reps=10):
        ctx.profile(True)
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
        rep = ctx.profile_report()
        ctx.profile(False)
        return {k: v[1] / v[0] for k, v in rep.items()}          # ms per launch

    d_desc, d_n = torch.from_numpy(desc).to(dev), torch.from_numpy(n).to(dev)
    torch.cuda.synchronize()
    o_syn, call_syn = dev_buffers(d_desc, d_n, nf, cap)

    # real ORB descriptors: 64 rendered frames, tiled to the batch size
    n_orb = 64
    oc = Context(640, 480, n_orb, nfeatures=1000)
    oc.set_stream(stream.cuda_stream)
    capk = int(oc.L.pslam_orb_max_keypoints(oc.h))
    frames = np.stack([synth.render_frame(3, k, 640, 480)[0] for k in range(n_orb)])
    g = torch.from_numpy(frames).to(dev)
    kps, od, on = (torch.empty((n_orb, capk, 28), dtype=torch.uint8, device=dev), torch.empty((n_orb, capk, 32), dtype=torch.uint8, device=dev),
                   torch.zeros(n_orb, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()
    oc.check(oc.L.pslam_orb_extract_batch_dev(oc.h, g.data_ptr(), n_orb, kps.data_ptr(), od.data_ptr(), capk, on.data_ptr()))
    torch.cuda.synchronize()
    reps = (nf + n_orb - 1) // n_orb
    d_desc_orb, d_n_orb = od.repeat(reps, 1, 1)[:nf].contiguous(), on.repeat(reps)[:nf].contiguous()
    torch.cuda.synchronize()
    o_orb, call_orb = dev_buffers(d_desc_orb, d_n_orb, nf, capk)
    res["orb_keypoints_mean"] = float(on.float().mean())

    # host-pointer batch call and the per-frame entry point
    h_out = dict(word_id=np.zeros((nf, cap), np.int32), word_val=np.zeros((nf, cap)), node_id=np.zeros((nf, cap), np.int32),
                 node_off=np.zeros((nf, cap + 1), np.int32), node_feat=np.zeros((nf, cap), np.int32))
    h_cnt = np.zeros((nf, 2), np.int32)
    host_call = lambda: ctx.check(L.pslam_bow_transform_batch(ctx.h, desc.ctypes.data, n.ctypes.data, cap, nf, 4, *[h_out[k].ctypes.data for k in KEYS],
                                                              h_cnt.ctypes.data))
    host_call()
    rounds = []
    for r in range(a.rounds):
        rd = {}
        rd["batch_dev_ms"] = float(np.median(time_dev(call_syn, a.iters)))
        rd["batch_dev_orb_ms"] = float(np.median(time_dev(call_orb, a.iters)))
        t = time.perf_counter()
        for _ in range(3):
            host_call()
        rd["batch_host_ms"] = (time.perf_counter() - t) * 1e3 / 3
        t = time.perf_counter()
        for f in range(3):
            bow_transform(ctx, voc, desc[f], 4)
        rd["single_frame_ms"] = (time.perf_counter() - t) * 1e3 / 3
        rounds.append(rd)
        print(f"round {r}: batch (device pointers) {rd['batch_dev_ms']:.3f} ms = {rd['batch_dev_ms'] * 1e3 / nf:.2f} us/frame; real ORB "
              f"{rd['batch_dev_orb_ms']:.3f} ms; host pointers {rd['batch_host_ms']:.1f} ms; per-frame pslam_bow_transform {rd['single_frame_ms']:.1f} ms/frame",
              flush=True)
    res["rounds"] = rounds
    res["kernels_synthetic_ms"] = kernel_split(call_syn)
    res["kernels_orb_ms"] = kernel_split(call_orb)
    print("kernel split (synthetic):", res["kernels_synthetic_ms"], "\nkernel split (ORB):", res["kernels_orb_ms"], flush=True)

    # outputs at the timed size against the CPU oracle
    bad = 0
    for f in np.random.default_rng(5).choice(nf, 8, replace=False):
        o = oracle_lib.bow_transform(voc, desc[f], 4)
        nw, nn = h_cnt[f]
        got = dict(word_id=h_out["word_id"][f, :nw], word_val=h_out["word_val"][f, :nw], node_id=h_out["node_id"][f, :nn], node_off=h_out["node_off"][f, :nn + 1],
                   node_feat=h_out["node_feat"][f, :h_out["node_off"][f, nn]])
        bad += any(got[k].tobytes() != o[k].tobytes() for k in KEYS)
    res["oracle_mismatching_frames_of_8"] = bad
    print(f"oracle check: {8 - bad} / 8 sampled frames identical", flush=True)

    if ref_lib.bow_lib() is not None:
        with tempfile.TemporaryDirectory() as td:
            path = os.path.join(td, "voc.txt")
            write_vocabulary_txt_fast(voc, path)
            t = time.perf_counter()
            rv = ref_lib.RefVocabulary(path)
            res["ref_load_s"] = time.perf_counter() - t
            m = 50
            t = time.perf_counter()
            for f in range(m):
                rv.transform(desc[f], 4)
            res["ref_ms_per_frame_1core"] = (time.perf_counter() - t) * 1e3 / m
            ncpu = os.cpu_count() or 1
            t = time.perf_counter()
            with cf.ThreadPoolExecutor(ncpu) as ex:                  # ctypes releases the GIL; transform() is const
                list(ex.map(lambda f: rv.transform(desc[f], 4), range(nf)))
            res["ref_batch_ms_all_cores"] = (time.perf_counter() - t) * 1e3
            res["host_cores"] = ncpu
            print(f"reference DBoW2: loadFromTextFile {res['ref_load_s']:.1f} s, {res['ref_ms_per_frame_1core']:.2f} ms/frame on one core, "
                  f"{res['ref_batch_ms_all_cores']:.0f} ms for {nf} frames on {ncpu} threads", flush=True)
    else:
        print("reference DBoW2: oracle/_ref/libbow_ref.so not present", flush=True)

    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
