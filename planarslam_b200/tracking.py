"""Host-side mirror of the device-resident tracking chain (include/pslam_abi.h pslam_track_*): Tracking::TrackWithMotionModel + TrackLocalMap
(src/Tracking.cc:1739-1859, 1954-2046) of a replayed RGB-D sequence against a POD map snapshot, without host round trips between stages or frames."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import Context


class TrackParams(C.Structure):
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("bf", C.c_float), ("depth_factor", C.c_float),
                ("min_x", C.c_float), ("max_x", C.c_float), ("min_y", C.c_float), ("max_y", C.c_float), ("th_last", C.c_float), ("th_map", C.c_float),
                ("nnratio_map", C.c_float), ("use_motion_model", C.c_int32)]


class MapPointsC(C.Structure):
    _fields_ = [("n", C.c_int32), ("pos", C.c_void_p), ("normal", C.c_void_p), ("max_distance", C.c_void_p), ("min_distance", C.c_void_p),
                ("desc", C.c_void_p), ("skip", C.c_void_p), ("has_obs", C.c_void_p)]


def default_params(K=(535.4, 539.2, 320.1, 247.6), bf=40.0, depth_factor=1.0 / 5000.0, width=640, height=480, use_motion_model=True) -> TrackParams:
    return TrackParams(K[0], K[1], K[2], K[3], bf, np.float32(depth_factor), 0.0, float(width), 0.0, float(height), 15.0, 3.0, 0.8, int(use_motion_model))


class Tracker:
    """tracker = Tracker(ctx); tracker.set_map(map_points_dict); poses, stats = tracker.track(gray [n,H,W] u8, depth [n,H,W] u16, Tcw0)"""

    def __init__(self, ctx: Context, params: TrackParams | None = None):
        self.ctx, self.params = ctx, params or default_params(width=ctx.cfg.width, height=ctx.cfg.height)
        L = ctx.L
        L.pslam_track_set_map.argtypes = [C.c_void_p, C.c_void_p]
        L.pslam_track_sequence.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        self._keep = None

    def set_map(self, m: dict):
        a = {k: np.ascontiguousarray(m[k], dt) for k, dt in (("pos", np.float32), ("normal", np.float32), ("max_distance", np.float32), ("min_distance", np.float32),
                                                             ("desc", np.uint8), ("skip", np.uint8), ("has_obs", np.uint8))}
        s = MapPointsC(len(a["skip"]), *[a[k].ctypes.data for k in ("pos", "normal", "max_distance", "min_distance", "desc", "skip", "has_obs")])
        self._keep = a
        self.ctx.check(self.ctx.L.pslam_track_set_map(self.ctx.h, C.byref(s)))

    def track(self, gray: np.ndarray, depth: np.ndarray, Tcw0: np.ndarray):
        g, d = np.ascontiguousarray(gray, np.uint8), np.ascontiguousarray(depth, np.uint16)
        n = len(g)
        T0 = np.ascontiguousarray(Tcw0, np.float32)
        poses, stats = np.zeros((n, 4, 4), np.float32), np.zeros((n, 4), np.int32)
        self.ctx.check(self.ctx.L.pslam_track_sequence(self.ctx.h, g.ctypes.data, d.ctypes.data, n, C.byref(self.params), T0.ctypes.data, poses.ctypes.data,
                                                       stats.ctypes.data))
        return poses, stats


class MapLinesC(C.Structure):
    _fields_ = [("n", C.c_int32), ("pos", C.c_void_p), ("normal", C.c_void_p), ("max_distance", C.c_void_p), ("min_distance", C.c_void_p),
                ("desc", C.c_void_p), ("skip", C.c_void_p), ("has_obs", C.c_void_p)]


class MapPlanesC(C.Structure):
    _fields_ = [("n", C.c_int32), ("coef", C.c_void_p), ("bad", C.c_void_p), ("pts_off", C.c_void_p), ("pts", C.c_void_p)]


class PlanarMapC(C.Structure):
    _fields_ = [("points", MapPointsC), ("lines", MapLinesC), ("planes", MapPlanesC), ("n_ref_lines", C.c_int32), ("ref_line_desc", C.c_void_p),
                ("ref_line_map", C.c_void_p), ("R_cm", C.c_float * 9)]


class PlanarTrackParams(C.Structure):
    _fields_ = [("base", TrackParams), ("line_th", C.c_float), ("line_nnratio", C.c_float), ("plane_dist_ref", C.c_float), ("plane_ang_ref", C.c_float),
                ("plane_ver_th", C.c_float), ("plane_par_th", C.c_float), ("angle_info", C.c_double), ("dist_info", C.c_double), ("par_info", C.c_double),
                ("ver_info", C.c_double), ("plane_chi", C.c_double), ("vp_chi", C.c_double), ("plane_dist_th", C.c_float), ("max_lines", C.c_int32),
                ("line_seed", C.c_uint32)]


PLANAR_STATS = 13      # PSLAM_PLANAR_STATS
PLANAR_STATS_FIELDS = ("mm_points", "mm_lines", "mm_planes", "mm_fallback", "mm_map_inliers", "mm_ok",
                       "lm_points", "lm_lines", "lm_planes", "lm_parallel", "lm_vertical", "lm_inliers", "lm_ok")


def default_planar_params(width=640, height=480, **kw) -> PlanarTrackParams:
    """TUM3.yaml: Plane.AssociationDisRef 0.05, AssociationAngRef 0.985, VerticalThreshold 0.08716, ParallelThreshold 0.98481, DistanceThreshold 0.05;
    the pose-optimisation plane settings of synth_pose.PLANE_SETTINGS; 40 key lines, srand seed 1."""
    from .synth_pose import PLANE_SETTINGS
    p = PlanarTrackParams(default_params(width=width, height=height), 1.0, 0.6, 0.05, 0.985, 0.08716, 0.98481, PLANE_SETTINGS["angle_info"],
                          PLANE_SETTINGS["dist_info"], PLANE_SETTINGS["par_info"], PLANE_SETTINGS["ver_info"], PLANE_SETTINGS["plane_chi"], PLANE_SETTINGS["vp_chi"],
                          0.05, 40, 1)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


class PlanarTracker:
    """PlanarSLAM's Tracking::Track() on the device (include/pslam_abi.h pslam_track_planar_*): Manhattan rotation, translation-only motion model, local map
    with point, line and plane edges.  tracker = PlanarTracker(ctx); tracker.set_map(planar_map_dict) (synth_planar_map.build_planar_map shows the keys);
    poses, Rcm, stats = tracker.track(gray [n,H,W] u8, depth [n,H,W] u16, Tcw0, vel0=None, Rcm0=None) - Rcm0 (mLastRcm before frame 0) defaults to
    R_cw(Tcw0) * Rotation_cm, the Manhattan frame seen from the start pose.
    update_map_planes: MapPlane::UpdateCoefficientsAndPoints after every frame, the clouds carried from call to call.  It is a setting of the context: the
    property reads it back from there, and the constructor changes it only when given True or False (None keeps it).  map_planes() returns the current
    clouds, plane_matches() each frame's final plane associations of the last call in that mode."""

    def __init__(self, ctx: Context, params: PlanarTrackParams | None = None, update_map_planes: bool | None = None):
        self.ctx, self.params = ctx, params or default_planar_params(width=ctx.cfg.width, height=ctx.cfg.height)
        L = ctx.L
        L.pslam_track_set_planar_map.argtypes = [C.c_void_p, C.c_void_p]
        L.pslam_track_planar_sequence.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p] + [C.c_void_p] * 6
        L.pslam_track_planar_set_map_plane_updates.argtypes = [C.c_void_p, C.c_int]
        L.pslam_track_planar_get_map_plane_updates.argtypes = [C.c_void_p]
        L.pslam_track_planar_map_planes.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.pslam_track_planar_plane_matches.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        self._keep, self.R_cm, self._n_planes, self._n_upload, self._last_n = None, None, 0, 0, 0
        if update_map_planes is not None:
            self.update_map_planes = update_map_planes

    @property
    def update_map_planes(self) -> bool:
        rc = self.ctx.L.pslam_track_planar_get_map_plane_updates(self.ctx.h)
        self.ctx.check(min(rc, 0))
        return rc == 1

    @update_map_planes.setter
    def update_map_planes(self, on: bool):
        self.ctx.check(self.ctx.L.pslam_track_planar_set_map_plane_updates(self.ctx.h, 1 if on else 0))

    def set_map(self, m: dict):
        f32, f64, u8, i32 = np.float32, np.float64, np.uint8, np.int32
        pt = {k: np.ascontiguousarray(m["points"][k], dt) for k, dt in (("pos", f32), ("normal", f32), ("max_distance", f32), ("min_distance", f32), ("desc", u8),
                                                                         ("skip", u8), ("has_obs", u8))}
        ln = {k: np.ascontiguousarray(m["lines"][k], dt) for k, dt in (("pos", f64), ("normal", f64), ("max_distance", f32), ("min_distance", f32), ("desc", u8),
                                                                        ("skip", u8), ("has_obs", u8))}
        pl = {k: np.ascontiguousarray(m["planes"][k], dt) for k, dt in (("coef", f32), ("bad", u8), ("pts_off", i32), ("pts", f32))}
        ref = {k: np.ascontiguousarray(m[k], dt) for k, dt in (("ref_line_desc", u8), ("ref_line_map", i32))}
        s = PlanarMapC()
        s.points = MapPointsC(len(pt["skip"]), *[pt[k].ctypes.data for k in ("pos", "normal", "max_distance", "min_distance", "desc", "skip", "has_obs")])
        s.lines = MapLinesC(len(ln["skip"]), *[ln[k].ctypes.data for k in ("pos", "normal", "max_distance", "min_distance", "desc", "skip", "has_obs")])
        s.planes = MapPlanesC(len(pl["bad"]), *[pl[k].ctypes.data for k in ("coef", "bad", "pts_off", "pts")])
        s.n_ref_lines, s.ref_line_desc, s.ref_line_map = len(ref["ref_line_map"]), ref["ref_line_desc"].ctypes.data, ref["ref_line_map"].ctypes.data
        self.R_cm = np.ascontiguousarray(m["R_cm"], np.float32).reshape(3, 3)
        s.R_cm[:] = [float(v) for v in self.R_cm.ravel()]
        self._keep = (pt, ln, pl, ref)
        self.ctx.check(self.ctx.L.pslam_track_set_planar_map(self.ctx.h, C.byref(s)))
        self._n_planes, self._n_upload = len(pl["bad"]), len(pl["pts"])

    def track(self, gray: np.ndarray, depth: np.ndarray, Tcw0: np.ndarray, vel0: np.ndarray | None = None, Rcm0: np.ndarray | None = None):
        g, d = np.ascontiguousarray(gray, np.uint8), np.ascontiguousarray(depth, np.uint16)
        n = len(g)
        T0 = np.ascontiguousarray(Tcw0, np.float32)
        v0 = None if vel0 is None else np.ascontiguousarray(vel0, np.float32)
        if Rcm0 is None:
            Rcm0 = (T0[:3, :3].astype(np.float64) @ self.R_cm.astype(np.float64)).astype(np.float32)
        R0 = np.ascontiguousarray(Rcm0, np.float32)
        poses, Rcm, stats = np.zeros((n, 4, 4), np.float32), np.zeros((n, 3, 3), np.float32), np.zeros((n, PLANAR_STATS), np.int32)
        self.ctx.check(self.ctx.L.pslam_track_planar_sequence(self.ctx.h, g.ctypes.data, d.ctypes.data, n, C.byref(self.params), T0.ctypes.data,
                                                              None if v0 is None else v0.ctypes.data, R0.ctypes.data, poses.ctypes.data, Rcm.ctypes.data,
                                                              stats.ctypes.data))
        self._last_n = n
        return poses, Rcm, stats

    def map_planes(self):
        """The map planes' current MapPlane::mvPlanePoints in upload order: (pts_off int32 [n + 1], pts float32 [pts_off[n]][3])."""
        off = np.zeros(self._n_planes + 1, np.int32)
        pts = np.zeros((max(self._n_planes * self.ctx.L.pslam_map_plane_max_points(self.ctx.h), self._n_upload), 3), np.float32)
        self.ctx.check(self.ctx.L.pslam_track_planar_map_planes(self.ctx.h, off.ctypes.data, pts.ctypes.data, len(pts)))
        return off, pts[:off[-1]].copy()

    def plane_matches(self, nframes: int | None = None) -> np.ndarray:
        """Each frame's final plane associations from the last track() with update_map_planes: int32 [nframes][3][maxp] = mvpMapPlanes,
        mvpParallelPlanes, mvpVerticalPlanes (map plane index or -1)."""
        n = self._last_n if nframes is None else nframes
        out = np.zeros((n, 3, self.ctx.L.pslam_peac_max_planes(self.ctx.h)), np.int32)
        self.ctx.check(self.ctx.L.pslam_track_planar_plane_matches(self.ctx.h, out.ctypes.data, n))
        return out
