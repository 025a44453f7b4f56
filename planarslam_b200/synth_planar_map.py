"""Synthetic planar map snapshot for the planar tracking chain (pslam_track_set_planar_map): map points, map lines, map planes, the reference key frame's
lines and Rotation_cm, built from the key frames of the three-plane room corner (synth.render_frame(2, f)) at their true poses with the Frame constructor's
products (pslam_frame_construct_batch)."""
from __future__ import annotations

import numpy as np

from . import synth, synth_map
from .frame import ConstructFrames


def build_planar_map(ctx, key_frames, seed: int = 2, n_frames: int = 64, max_lines: int = 40) -> dict:
    """key_frames: frame indices; the last one is the reference key frame.  Points as synth_map.map_from_frame; lines from the lines isLineGood accepted,
    world end points Twc * mvLines3D with MapLine's normal and distances (src/MapLine.cpp:44-55); planes pi_w = Tcw^T pi_c of ComputePlanes' coefficients with
    the voxel points in world coordinates; Rotation_cm from the first key frame's three planes, in world coordinates."""
    frames = [synth.render_frame(seed, f, n_frames=n_frames)[:2] for f in key_frames]
    out = ConstructFrames(ctx, np.stack([g for g, _ in frames]), np.stack([d for _, d in frames]), line_seed=1)
    pts, lines, planes, ref = [], [], [], None
    for k, f in enumerate(key_frames):
        Tcw = synth_map.true_pose(f, n_frames)
        nk = int(out.n_keys[k])
        fa = synth_map.frame_arrays(out.keys[k, :nk], out.desc[k, :nk], frames[k][1])
        pts.append(synth_map.map_from_frame(fa, Tcw))
        R, t = Tcw[:3, :3], Tcw[:3, 3]
        Ow = -R.T @ t
        nl = int(out.n_lines[k])
        l3 = out.lines3d[k, :nl]
        base = sum(len(x["skip"]) for x in lines)
        ref_map = np.full(nl, -1, np.int32)
        L = dict(pos=[], normal=[], max_distance=[], min_distance=[], desc=[], skip=[], has_obs=[])
        for i in range(nl):
            if not l3["valid"][i]:
                continue
            A, B = R.T @ (l3["A"][i] - t), R.T @ (l3["B"][i] - t)
            PC = 0.5 * (A + B) - Ow
            dist = np.float32(np.linalg.norm(PC))
            maxd = np.float32(dist * synth_map.SCALE_FACTORS[out.keylines[k, i]["octave"]])
            ref_map[i] = base + len(L["skip"])
            L["pos"].append(np.concatenate([A, B])); L["normal"].append(PC / np.linalg.norm(PC)); L["max_distance"].append(maxd)
            L["min_distance"].append(np.float32(maxd / synth_map.SCALE_FACTORS[-1])); L["desc"].append(out.line_desc[k, i]); L["skip"].append(0); L["has_obs"].append(1)
        lines.append({key: np.array(v).reshape(len(v), -1) if key in ("pos", "normal", "desc") else np.array(v) for key, v in L.items()})
        ref = dict(ref_line_desc=np.ascontiguousarray(out.line_desc[k, :nl]), ref_line_map=ref_map)
        T32 = Tcw.astype(np.float32)
        for p in range(int(out.n_planes[k])):
            c = out.plane_coef[k, p].astype(np.float64)
            pw = (T32.astype(np.float64).T @ c).astype(np.float32)
            a, b = out.plane_pt_off[k, p], out.plane_pt_off[k, p + 1]
            P = out.plane_pts[k, a:b].astype(np.float64)
            planes.append((pw, ((P - t) @ R).astype(np.float32)))
    cat = lambda parts, key, dt: np.concatenate([np.asarray(x[key], dt).reshape(len(x["skip"]), -1) if np.asarray(x[key]).ndim > 1 or key in ("pos", "normal", "desc")
                                                 else np.asarray(x[key], dt) for x in parts if len(x["skip"])])
    point_keys = (("pos", np.float32), ("normal", np.float32), ("max_distance", np.float32), ("min_distance", np.float32), ("desc", np.uint8), ("skip", np.uint8),
                  ("has_obs", np.uint8))
    P = {key: cat(pts, key, dt) for key, dt in point_keys}
    P["pos"], P["normal"], P["desc"] = P["pos"].reshape(-1, 3), P["normal"].reshape(-1, 3), P["desc"].reshape(-1, 32)
    Lm = {key: cat(lines, key, dt) for key, dt in (("pos", np.float64), ("normal", np.float64), ("max_distance", np.float32), ("min_distance", np.float32),
                                                   ("desc", np.uint8), ("skip", np.uint8), ("has_obs", np.uint8))}
    Lm["pos"], Lm["normal"], Lm["desc"] = Lm["pos"].reshape(-1, 6), Lm["normal"].reshape(-1, 3), Lm["desc"].reshape(-1, 32)
    off = np.zeros(len(planes) + 1, np.int32)
    off[1:] = np.cumsum([len(p[1]) for p in planes])
    Pl = dict(coef=np.array([p[0] for p in planes], np.float32).reshape(-1, 4), bad=np.zeros(len(planes), np.uint8), pts_off=off,
              pts=np.concatenate([p[1] for p in planes]).astype(np.float32).reshape(-1, 3) if planes else np.zeros((0, 3), np.float32))
    # Rotation_cm: the Manhattan axes in the map (world) frame - the normals of the first key frame's three largest planes, projected onto SO(3) and
    # rotated into the world; R_cw * Rotation_cm is then the mLastRcm of a camera at pose R_cw
    N = out.plane_coef[0, :3, :3].astype(np.float64).T
    U, _, Vt = np.linalg.svd(N)
    Rc = U @ Vt
    if np.linalg.det(Rc) < 0:
        Rc[:, 2] = -Rc[:, 2]
    R_cm = (synth_map.true_pose(key_frames[0], n_frames)[:3, :3].T @ Rc).astype(np.float32)
    return dict(points=P, lines=Lm, planes=Pl, R_cm=R_cm, **ref)
