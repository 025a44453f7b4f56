"""GPU: the device-resident planar tracking chain (pslam_track_planar_sequence, PlanarSLAM's Tracking::Track()) on the synthetic room corner, against THE SAME
CHAIN COMPOSED FROM THE REFERENCE'S OWN FUNCTIONS on the CPU: Tracking::TrackManhattanFrame (libtrack_ref), ORBmatcher::SearchByProjection x2,
LSDmatcher::SearchByDescriptor, Frame::isInFrustum(MapLine*) + LSDmatcher::SearchByProjection, PlaneMatcher::SearchMapByCoefficients, Optimizer::
TranslationOptimization / PoseOptimization (libmatch_ref: src/*.cc and Thirdparty/g2o compiled unmodified); MatchORBPoints from the cv2-pinned matcher
oracle.  Only the glue is numpy: the gates, the sweeps, the pose and rotation products in float storage / double accumulation, with the conventions of
include/pslam_abi.h.  Per-frame inputs come from pslam_frame_construct_batch (checked against the oracles elsewhere), so the test isolates the orchestration.
Falls back to the oracle restatements of the same functions when oracle/_ref is absent."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib
import ref_lib
from planarslam_b200 import synth, synth_map, synth_pose
from planarslam_b200._lib import Context, PslamError
from planarslam_b200.frame import ConstructFrames
from planarslam_b200.synth_planar_map import build_planar_map
from planarslam_b200.tracking import PLANAR_STATS_FIELDS, PlanarTracker, Tracker, default_planar_params

pytestmark = pytest.mark.gpu
N_FRAMES = 64
F = {k: i for i, k in enumerate(PLANAR_STATS_FIELDS)}


def _mm(a, b):
    return (np.asarray(a, np.float64) @ np.asarray(b, np.float64)).astype(np.float32)


def _inv_pose(T):
    R, t = T[:3, :3], T[:3, 3]
    out = np.eye(4, dtype=np.float32)
    out[:3, :3] = R.T
    out[:3, 3] = (-(R.T.astype(np.float64)) @ t.astype(np.float64)).astype(np.float32)
    return out


class _Ref:
    """The reference's functions (or their oracle restatements when oracle/_ref is absent)."""

    def __init__(self):
        self.use_ref = ref_lib.match_lib() is not None and ref_lib.track_lib() is not None
        self.L = oracle_lib.lib()

    def manhattan(self, R, normals, dirs):
        return ref_lib.ref_track_manhattan_frame(R, normals, dirs) if self.use_ref else oracle_lib.track_manhattan_frame(R, normals, dirs)["R"]

    def search_last(self, *a):
        return (ref_lib.ref_search_by_projection_last if self.use_ref else oracle_lib.search_by_projection_last)(*a)

    def search_map(self, *a):
        return (ref_lib.ref_search_by_projection_map if self.use_ref else oracle_lib.search_by_projection_map)(*a)

    def lines_in_frustum(self, *a):
        return (ref_lib.ref_lines_in_frustum if self.use_ref else oracle_lib.lines_in_frustum)(*a)

    def line_search(self, *a):
        return (ref_lib.ref_line_search_by_projection if self.use_ref else oracle_lib.line_search_by_projection)(*a)

    def optimise(self, p, translation_only):
        return ref_lib.ref_full_pose_optimization(p, translation_only) if self.use_ref else oracle_lib.pose_optimization(p, translation_only)

    def knn2(self, q, t):
        L = self.L
        L.orc_bf_knn2.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        q, t = np.ascontiguousarray(q, np.uint8), np.ascontiguousarray(t, np.uint8)
        idx, dist = np.zeros((max(len(q), 1), 2), np.int32), np.zeros((max(len(q), 1), 2), np.int32)
        L.orc_bf_knn2(q.ctypes.data, len(q), t.ctypes.data, len(t), idx.ctypes.data, dist.ctypes.data)
        return idx[:len(q)], dist[:len(q)]

    def match_orb_points(self, cur_desc, last_desc, m_last, o_last):
        """ORBmatcher::MatchORBPoints (src/ORBmatcher.cc:1332-1394) with cv::BFMatcher::match and its gate from the cv2-pinned oracle; the
        mvbOutlier[i] index quirk kept.  Returns (NPair, matches)."""
        matches = np.full(len(cur_desc), -1, np.int32)
        if len(cur_desc) == 0 or len(last_desc) == 0:
            return 0, matches
        idx, dist = self.knn2(cur_desc, last_desc)
        self.L.orc_match_gate.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        d1 = np.ascontiguousarray(dist[:, 0])
        keep = np.zeros(len(cur_desc), np.int32)
        n = self.L.orc_match_gate(d1.ctypes.data, len(cur_desc), keep.ctypes.data)
        for k, qi in enumerate(keep[:n]):
            mp = m_last[idx[qi, 0]]
            if mp >= 0 and not (k < len(o_last) and o_last[k]):
                matches[qi] = mp
        return n, matches

    def line_search_by_descriptor(self, ref_desc, ref_map, f_desc):
        """LSDmatcher::SearchByDescriptor(mpReferenceKF, cur): (nmatches, map line per frame line).  Fewer than two frame lines: no match (the reference
        reads a second neighbour that knnMatch did not return)."""
        if len(f_desc) < 2 or len(ref_desc) == 0:
            return 0, np.full(len(f_desc), -1, np.int32)
        if self.use_ref:
            n, q = ref_lib.ref_line_search_by_descriptor(ref_desc, (ref_map >= 0).astype(np.uint8), f_desc)
        else:
            idx, dist = self.knn2(ref_desc, f_desc)
            q, n = np.full(len(f_desc), -1, np.int32), 0
            for i in range(len(ref_desc)):
                with np.errstate(divide="ignore", invalid="ignore"):
                    ratio = np.float32(dist[i, 0]) / np.float32(dist[i, 1])
                if float(ratio) < float(np.float32(1.0) / np.float32(1.5)) and ref_map[i] >= 0:
                    q[idx[i, 0]] = i
                    n += 1
        return n, np.where(q >= 0, ref_map[np.maximum(q, 0)], -1).astype(np.int32)

    def plane_match(self, T, fc, P, prm):
        a = (T, fc, P["coef"], P["bad"], P["pts_off"], P["pts"], prm.plane_dist_ref, prm.plane_ang_ref, prm.plane_ver_th, prm.plane_par_th)
        if self.use_ref:
            n, om, ov, op = ref_lib.ref_plane_match(*a)
        else:
            L = self.L
            L.orc_plane_match.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_float] * 4 + \
                [C.c_void_p] * 3
            T, fc2 = np.ascontiguousarray(T, np.float32), np.ascontiguousarray(fc, np.float32)
            om, ov, op = [np.full(max(len(fc), 1), -1, np.int32) for _ in range(3)]
            n = L.orc_plane_match(T.ctypes.data, len(fc), fc2.ctypes.data, len(P["bad"]), P["coef"].ctypes.data, P["bad"].ctypes.data, P["pts_off"].ctypes.data,
                                  P["pts"].ctypes.data, *a[6:], om.ctypes.data, ov.ctypes.data, op.ctypes.data)
            om, ov, op = om[:len(fc)], ov[:len(fc)], op[:len(fc)]
        return n, np.stack([om, op, ov]) if len(fc) else np.zeros((3, 0), np.int32)      # [mvpMapPlanes, mvpParallelPlanes, mvpVerticalPlanes]


def _problem(fa, matches, lmatch, lf, mp3, fc, m, T, mode):
    """What Optimizer::PoseOptimization (mode 0) / TranslationOptimization (mode 1) reads from the Frame: points, lines, planes (and parallel / vertical
    planes in mode 0) in frame order."""
    P, Lm, Pl = m["points"], m["lines"], m["planes"]
    idx = np.nonzero(matches >= 0)[0]
    k = fa["keys_un"][idx]
    inv_sigma2 = (np.float32(1.0) / (synth_map.SCALE_FACTORS ** 2).astype(np.float32)).astype(np.float32)
    lidx = np.nonzero(lmatch >= 0)[0]
    fam = [np.nonzero(mp3[f] >= 0)[0] for f in range(3)]
    if mode == 1:
        fam = [fam[0], fam[1][:0], fam[2][:0]]
    meas = [np.ascontiguousarray(fc[fam[f]], np.float32).reshape(-1, 4) for f in range(3)]
    mapp = [np.ascontiguousarray(Pl["coef"][mp3[f][fam[f]]], np.float32).reshape(-1, 4) for f in range(3)]
    p = dict(fx=synth.TUM3_K[0], fy=synth.TUM3_K[1], cx=synth.TUM3_K[2], cy=synth.TUM3_K[3], bf=40.0, Xw=np.ascontiguousarray(P["pos"][matches[idx]], np.float32),
             obs=np.ascontiguousarray(np.stack([k["x"], k["y"], fa["u_right"][idx]], 1), np.float32), inv_sigma2=np.ascontiguousarray(inv_sigma2[k["octave"]]),
             line_Xw=np.ascontiguousarray(Lm["pos"][lmatch[lidx]], np.float64).reshape(-1, 6), line_obs=np.ascontiguousarray(lf[lidx], np.float64).reshape(-1, 3),
             plane_meas=meas[0], plane_map=mapp[0], par_meas=meas[1], par_map=mapp[1], ver_meas=meas[2], ver_map=mapp[2],
             Tcw0=np.ascontiguousarray(T, np.float32), **synth_pose.PLANE_SETTINGS)
    return p, idx, lidx, fam


def _reference_chain(fr, m, T0, prm):
    """Tracking::Track() per frame, composed from the reference's functions (include/pslam_abi.h conventions).  fr: FrameOutputs of the sequence.
    Returns poses, mLastRcm, stats rows, line / plane inliers of the local-map stage."""
    R = _Ref()
    P, Lm, Pl = m["points"], m["lines"], m["planes"]
    pts_map = dict(n=len(P["skip"]), **{k: np.ascontiguousarray(v) for k, v in P.items()})
    ref_desc, ref_map = np.ascontiguousarray(m["ref_line_desc"], np.uint8), np.asarray(m["ref_line_map"], np.int32)
    R_cm = np.asarray(m["R_cm"], np.float32)
    T = np.ascontiguousarray(T0, np.float32)
    Rcm = _mm(T[:3, :3], R_cm)
    vel = np.eye(4, dtype=np.float32)
    poses, rcms, stats, lin, pin = [], [], [], [], []
    fa_prev = m_prev = o_prev = None
    for t in range(fr.nframes):
        nk, nl, npl = int(fr.n_keys[t]), int(fr.n_lines[t]), int(fr.n_planes[t])
        fa = dict(n=nk, keys_un=np.ascontiguousarray(fr.keys[t, :nk]), u_right=np.ascontiguousarray(fr.u_right[t, :nk]), desc=np.ascontiguousarray(fr.desc[t, :nk]))
        kl, lf, ld, l3 = fr.keylines[t, :nl], fr.line_functions[t, :nl], np.ascontiguousarray(fr.line_desc[t, :nl]), fr.lines3d[t, :nl]
        fc = np.ascontiguousarray(fr.plane_coef[t, :npl], np.float32)
        MF = R.manhattan(Rcm, fr.surface_normals8[t][:, :3], l3["director"][l3["valid"] != 0])
        Rcm = MF
        st = np.zeros(13, np.int32)
        matches, outl, lmatch = np.full(nk, -1, np.int32), np.zeros(nk, np.uint8), np.full(nl, -1, np.int32)
        mp3 = np.full((3, npl), -1, np.int32)
        skip, lskip = P["skip"].copy(), Lm["skip"].copy()
        on, ok = True, False
        n_line_in = n_plane_in = 0
        if t > 0:
            last = T
            T = _mm(vel, last)
            pred = T.copy()
            Rcw = _mm(R_cm, MF.T).T
            lfr = dict(n=fa_prev["n"], keys=fa_prev["keys_un"], map_point=m_prev, outlier=o_prev, Tcw=last)
            n, matches = R.search_last(synth_map.frame_view(fa, T), lfr, pts_map, 15.0, False, True, matches)
            matches = matches.copy()
            if n < 50:
                st[3] = 1
                n, matches = R.match_orb_points(fa["desc"], fa_prev["desc"], m_prev, o_prev)
            ln, lmatch = R.line_search_by_descriptor(ref_desc, ref_map, ld)
            pn, f3 = R.plane_match(T, fc, Pl, prm)
            mp3 = np.where(f3 >= 0, f3, mp3)
            st[0:3] = n, ln, pn
            if n + ln + pn < 10:
                T, on = pred, False
            else:
                T = T.copy()
                T[:3, :3] = Rcw
                p, idx, lidx, fam = _problem(fa, matches, lmatch, lf, mp3, fc, m, T, 1)
                r = R.optimise(p, True) if len(idx) >= 3 else None
                fo = lambda key, k: r is not None and r[key][k] != 0
                n_map = n_l = n_p = 0
                for k, i in enumerate(idx):
                    if fo("outlier_pt", k):
                        skip[matches[i]] = 1
                        matches[i] = -1
                    elif P["has_obs"][matches[i]]:
                        n_map += 1
                for k, i in enumerate(lidx):
                    if fo("outlier_line", k):
                        lskip[lmatch[i]] = 1
                        lmatch[i] = -1
                    elif Lm["has_obs"][lmatch[i]]:
                        n_l += 1
                for k, i in enumerate(fam[0]):
                    n_p += not fo("outlier_plane", k)
                if r is not None:
                    T = np.ascontiguousarray(r["Tcw"], np.float32)
                ok_mm = not (n_map < 3 or n_map + n_l + n_p < 3)
                st[4], st[5] = n_map, ok_mm
                if not ok_mm:
                    T, on = pred, False
        if on:
            skip[matches[matches >= 0]] = 1
            _, matches, _ = R.search_map(synth_map.frame_view(fa, T), dict(pts_map, skip=skip), 3.0, 0.8, matches)
            matches = matches.copy()
            lskip[lmatch[lmatch >= 0]] = 1
            if len(Lm["skip"]):
                fv = synth_map.frame_view(fa, T)
                o = R.lines_in_frustum(fv, Lm["pos"], Lm["normal"], Lm["max_distance"], Lm["min_distance"], 0.6)
                in_view = (o["in_view"] != 0) & (lskip == 0)
                occ = np.array([lm >= 0 and Lm["has_obs"][lm] for lm in lmatch], np.uint8)
                frame = dict(pt=np.ascontiguousarray(kl["pt"], np.float32), angle=np.ascontiguousarray(kl["angle"]), octave=np.ascontiguousarray(kl["octave"]),
                             desc=ld, has_obs=occ, scale_factors=synth_map.SCALE_FACTORS)
                ml = dict(skip=(~in_view).astype(np.uint8), level=o["level"], view_cos=o["view_cos"], proj=o["proj"], desc=Lm["desc"], has_obs=Lm["has_obs"])
                if nl:
                    _, assigned = R.line_search(frame, ml, prm.line_th, prm.line_nnratio)
                    lmatch = np.where(assigned >= 0, assigned, lmatch).astype(np.int32)
            _, f3 = R.plane_match(T, fc, Pl, prm)
            mp3 = np.where(f3 >= 0, f3, mp3)
            p, idx, lidx, fam = _problem(fa, matches, lmatch, lf, mp3, fc, m, T, 0)
            n_init = len(idx) + len(lidx) + sum(len(f) for f in fam)
            r = R.optimise(p, False) if n_init >= 3 else None
            fo = lambda key, k: r is not None and r[key][k] != 0
            n_pt_in = 0
            for k, i in enumerate(idx):
                if fo("outlier_pt", k):
                    outl[i] = 1
                elif P["has_obs"][matches[i]]:
                    n_pt_in += 1
            n_line_in = sum(1 for k, i in enumerate(lidx) if not fo("outlier_line", k) and Lm["has_obs"][lmatch[i]])
            n_plane_in = sum(1 for k in range(len(fam[0])) if not fo("outlier_plane", k))
            if r is not None:
                T = np.ascontiguousarray(r["Tcw"], np.float32)
            inl = n_pt_in + n_line_in + n_plane_in
            ok = inl >= 7
            st[6:13] = len(idx), len(lidx), len(fam[0]), len(fam[1]), len(fam[2]), inl, ok
            if ok:
                drop = (matches >= 0) & (P["has_obs"][np.maximum(matches, 0)] == 0)
                matches[drop], outl[drop] = -1, 0
        if t > 0:
            if ok:
                vel = _mm(T, _inv_pose(last))
            Rcm = _mm(R_cm.T, T[:3, :3].T).T
        poses.append(T.copy()); rcms.append(Rcm.copy()); stats.append(st); lin.append(n_line_in); pin.append(n_plane_in)
        fa_prev, m_prev, o_prev = fa, matches, outl
    return np.stack(poses), np.stack(rcms), np.stack(stats), np.array(lin), np.array(pin)


def _compare(poses, Rcm, stats, ref, frames_ok=None):
    rp, rr, rs = ref[:3]
    worst = (0.0, 0.0, 0.0)
    for t in range(len(poses)):
        da, dt = synth_pose.pose_error(poses[t], rp[t])
        dr = float(np.abs(Rcm[t].astype(np.float64) - rr[t]).max())
        worst = (max(worst[0], da), max(worst[1], dt), max(worst[2], dr))
        assert da < 1e-4 and dt < 1e-3 and dr < 1e-4, (t, da, dt, dr, stats[t], rs[t])
    return worst


@pytest.fixture(scope="module")
def setup():
    ctx = Context(640, 480, max_batch=N_FRAMES)
    frames = [synth.render_frame(2, f)[:2] for f in range(N_FRAMES)]
    m = build_planar_map(ctx, list(range(0, N_FRAMES, 8)))
    return ctx, frames, m


def test_planar_chain_matches_the_reference_chain(setup):
    ctx, frames, m = setup
    gray, depth = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
    prm = default_planar_params()
    fr = ConstructFrames(ctx, gray, depth, depth_factor=prm.base.depth_factor, bf=prm.base.bf, plane_dist_th=prm.plane_dist_th, line_seed=prm.line_seed)
    T0 = synth_map.true_pose(0).astype(np.float32)
    ref = _reference_chain(fr, m, T0, prm)
    tr = PlanarTracker(ctx, prm)
    tr.set_map(m)
    poses, Rcm, stats = tr.track(gray, depth, T0)
    worst = _compare(poses, Rcm, stats, ref)
    for t in range(N_FRAMES):
        ea, et = synth_pose.pose_error(poses[t], synth_map.true_pose(t))
        assert ea < 5e-3 and et < 2e-2, (t, ea, et)
    assert np.mean(np.all(stats == ref[2], axis=1)) >= 0.8, (stats[:6], ref[2][:6])
    # the reference chain's local-map stage has line and plane inliers, so a fixture without them cannot pass
    assert np.mean(ref[3] > 0) >= 0.75 and np.mean(ref[4] > 0) >= 0.75, (ref[3], ref[4])
    assert (ref[2][:, F["lm_parallel"]] > 0).any() and (ref[2][:, F["lm_vertical"]] > 0).any()
    print("worst difference vs the reference chain (rad, m, mLastRcm):", worst, "frames with equal stats:", np.mean(np.all(stats == ref[2], axis=1)))


def test_planar_chain_tracks_the_room_corner(setup):
    ctx, frames, m = setup
    assert len(m["lines"]["skip"]) > 50 and len(m["planes"]["bad"]) >= 3
    tr = PlanarTracker(ctx)
    tr.set_map(m)
    T0 = synth_map.true_pose(0).astype(np.float32)
    poses, Rcm, stats = tr.track(np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames]), T0)
    for t in range(N_FRAMES):
        ea, et = synth_pose.pose_error(poses[t], synth_map.true_pose(t))
        assert ea < 5e-3 and et < 2e-2, (t, ea, et, stats[t])
        if t > 0:       # mLastRcm = (Rotation_cm^T R_cw^T)^T of the final pose (src/Tracking.cc:281-284)
            expect = _mm(m["R_cm"].T, poses[t][:3, :3].T).T
            assert np.abs(Rcm[t] - expect).max() < 1e-6, (t, Rcm[t], expect)
    assert (stats[1:, F["mm_ok"]] == 1).all() and (stats[:, F["lm_ok"]] == 1).all(), stats
    # lines and planes take part in the local-map optimisation on most frames (a map without them cannot pass)
    assert np.mean(stats[:, F["lm_lines"]] > 0) >= 0.75 and np.mean(stats[:, F["lm_planes"]] > 0) >= 0.75, stats[:, 6:11]
    assert np.mean(stats[1:, F["mm_lines"]] > 0) >= 0.75 and np.mean(stats[1:, F["mm_planes"]] > 0) >= 0.75, stats[:, :6]
    print("stats (first frames):", stats[:4])


def test_blank_frames_take_the_failure_path(setup):
    ctx, frames, m = setup
    n = 24
    gray, depth = np.stack([f[0] for f in frames[:n]]), np.stack([f[1] for f in frames[:n]])
    blank = list(range(10, 14))
    gray[blank] = 0
    depth[blank] = 0
    tr = PlanarTracker(ctx)
    tr.set_map(m)
    poses, Rcm, stats = tr.track(gray, depth, synth_map.true_pose(0).astype(np.float32))
    # the same flags, MatchORBPoints use and poses as the reference chain's glue under the documented conventions
    prm = default_planar_params()
    fr = ConstructFrames(ctx, gray, depth, depth_factor=prm.base.depth_factor, bf=prm.base.bf, plane_dist_th=prm.plane_dist_th, line_seed=prm.line_seed)
    ref = _reference_chain(fr, m, synth_map.true_pose(0).astype(np.float32), prm)
    for col in ("mm_ok", "lm_ok", "mm_fallback"):
        assert np.array_equal(stats[:, F[col]], ref[2][:, F[col]]), (col, stats[:, F[col]], ref[2][:, F[col]])
    _compare(poses, Rcm, stats, ref)
    for t in blank:
        assert stats[t, F["mm_ok"]] == 0 and stats[t, F["lm_ok"]] == 0, (t, stats[t])
        assert stats[t, F["mm_fallback"]] == 1 and (stats[t, 6:] == 0).all(), (t, stats[t])
    # a failed frame keeps mVelocity * mLastFrame.mTcw and leaves the velocity alone: the blank run extrapolates the last velocity
    vel = _mm(poses[9], np.linalg.inv(poses[8].astype(np.float64)).astype(np.float32))
    for t in blank:
        ea, et = synth_pose.pose_error(poses[t], _mm(vel, poses[t - 1]))
        assert ea < 1e-5 and et < 1e-5, (t, ea, et)
    assert (stats[:10, F["lm_ok"]] == 1).all()


def test_planar_argument_checks_and_the_points_chain_is_untouched(setup):
    ctx, frames, m = setup
    g, d = np.stack([f[0] for f in frames[:8]]), np.stack([f[1] for f in frames[:8]])
    T0 = synth_map.true_pose(0).astype(np.float32)
    fresh = Context(640, 480, max_batch=8)
    with pytest.raises(PslamError) as e:
        PlanarTracker(fresh).track(g, d, T0, Rcm0=m["R_cm"])
    assert e.value.code == -1                                    # PSLAM_E_INVALID: no planar map
    tr = PlanarTracker(fresh)
    tr.set_map(m)
    with pytest.raises(PslamError) as e:
        tr.track(np.concatenate([g, g[:1]]), np.concatenate([d, d[:1]]), T0)
    assert e.value.code == -1                                    # nframes > max_batch
    # the points-only chain: same result before and after a planar map upload
    ctx2 = Context(640, 480, max_batch=8)
    pts = dict(m["points"]); pts["n"] = len(pts["skip"])
    tk = Tracker(ctx2)
    tk.set_map(pts)
    p0, s0 = tk.track(g, d, T0)
    PlanarTracker(ctx2).set_map(m)
    p1, s1 = tk.track(g, d, T0)
    assert np.array_equal(p0, p1) and np.array_equal(s0, s1)
