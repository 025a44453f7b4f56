"""ctypes access to the CPU oracle (oracle/_build/liboracle.so). Test infrastructure only."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_PATH = os.path.join(ROOT, "oracle", "_build", "liboracle_fast.so" if os.environ.get("PSLAM_REF_VARIANT") == "fast" else "liboracle.so")   # fast: CPU-baseline build only
KEYPOINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                           ("octave", "<i4"), ("class_id", "<i4")])
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            subprocess.run(["make"] + (["fast"] if _PATH.endswith("_fast.so") else []), cwd=os.path.join(ROOT, "oracle"), check=True, stdout=subprocess.DEVNULL)
        L = C.CDLL(_PATH)
        vp, i = C.c_void_p, C.c_int
        L.orc_orb_create.restype = vp
        L.orc_orb_create.argtypes = [i, C.c_float, i, i, i]
        L.orc_orb_destroy.argtypes = [vp]
        L.orc_orb_extract.argtypes = [vp, vp, i, i, i, vp, vp, i]
        L.orc_orb_level_size.argtypes = [vp, i, C.POINTER(i), C.POINTER(i)]
        L.orc_orb_level_pixels.argtypes = [vp, i, vp]
        L.orc_orb_level_candidates.argtypes = [vp, i, vp, i]
        L.orc_orb_level_keypoints.argtypes = [vp, i, vp, i]
        L.orc_orb_tables.argtypes = [vp] + [vp] * 6
        L.orc_orb_describe.argtypes = [vp, vp, i, i, C.c_float, C.c_float, C.c_float, vp]
        L.orc_orb_ic_angle.argtypes = [vp, vp, i, i, i, i]
        L.orc_orb_ic_angle.restype = C.c_float
        L.orc_resize_linear_u8.argtypes = [vp, i, i, i, vp, i, i]
        L.orc_border_reflect101.argtypes = [vp, i, i, i, vp, i]
        L.orc_gaussian_blur_7x7_s2.argtypes = [vp, i, i, i, vp]
        L.orc_fast_detect.argtypes = [vp, i, i, i, i, vp, i]
        L.orc_fast_atan2.argtypes = [C.c_float, C.c_float]
        L.orc_fast_atan2.restype = C.c_float
        L.orc_cv_round.argtypes = [C.c_double]
        L.orc_peac_run.restype = vp
        L.orc_peac_run.argtypes = [vp, i, i] + [C.c_float] * 5
        L.orc_peac_free.argtypes = [vp]
        L.orc_peac_num_planes.argtypes = [vp]
        L.orc_peac_num_coarse.argtypes = [vp]
        L.orc_peac_labels.argtypes = [vp, vp]
        L.orc_peac_plane.argtypes = [vp, i, vp, vp]
        L.orc_peac_membership.argtypes = [vp, i, vp, i]
        L.orc_peac_blocks.argtypes = [vp, vp, vp]
        L.orc_peac_coarse_blocks.argtypes = [vp, vp]
        L.orc_eig33.argtypes = [vp, vp, vp]
        L.orc_heap_selftest.argtypes = [vp, i, vp, i]
        _lib = L
    return _lib


class OrbOracle:
    def __init__(self, nfeatures=1000, scale=1.2, nlevels=8, ini_th=20, min_th=7):
        self.L = lib()
        self.h = self.L.orc_orb_create(nfeatures, scale, nlevels, ini_th, min_th)
        self.nlevels = nlevels

    def __del__(self):
        if getattr(self, "h", None):
            self.L.orc_orb_destroy(self.h)
            self.h = None

    def extract(self, gray: np.ndarray):
        gray = np.ascontiguousarray(gray)
        h, w = gray.shape
        cap = 8192
        kps = np.zeros(cap, KEYPOINT_DTYPE)
        desc = np.zeros((cap, 32), np.uint8)
        n = self.L.orc_orb_extract(self.h, gray.ctypes.data, w, h, w, kps.ctypes.data, desc.ctypes.data, cap)
        assert n <= cap
        return kps[:n].copy(), desc[:n].copy()

    def level(self, l: int) -> np.ndarray:
        w, h = C.c_int(), C.c_int()
        assert self.L.orc_orb_level_size(self.h, l, C.byref(w), C.byref(h)) == 0
        out = np.zeros((h.value, w.value), np.uint8)
        self.L.orc_orb_level_pixels(self.h, l, out.ctypes.data)
        return out

    def candidates(self, l: int) -> np.ndarray:
        buf = np.zeros((200000, 3), np.int32)
        n = self.L.orc_orb_level_candidates(self.h, l, buf.ctypes.data, 200000)
        return buf[:n].copy()

    def level_keypoints(self, l: int) -> np.ndarray:
        buf = np.zeros(8192, KEYPOINT_DTYPE)
        n = self.L.orc_orb_level_keypoints(self.h, l, buf.ctypes.data, 8192)
        return buf[:n].copy()

    def tables(self):
        f = [np.zeros(self.nlevels, np.float32) for _ in range(4)]
        q = np.zeros(self.nlevels, np.int32)
        um = np.zeros(16, np.int32)
        self.L.orc_orb_tables(self.h, *[a.ctypes.data for a in f], q.ctypes.data, um.ctypes.data)
        return f + [q, um]


def orb_extract(gray, nfeatures=1000, scale=1.2, nlevels=8, ini_th=20, min_th=7):
    return OrbOracle(nfeatures, scale, nlevels, ini_th, min_th).extract(gray)


def blur(gray: np.ndarray) -> np.ndarray:
    gray = np.ascontiguousarray(gray)
    out = np.empty_like(gray)
    lib().orc_gaussian_blur_7x7_s2(gray.ctypes.data, gray.shape[1], gray.shape[0], gray.shape[1], out.ctypes.data)
    return out


class PeacOracle:
    """Result of the oracle PEAC on one depth image."""

    def __init__(self, depth: np.ndarray, K=(535.4, 539.2, 320.1, 247.6), scale=np.float32(1.0 / 5000.0)):
        L = lib()
        depth = np.ascontiguousarray(depth)
        h, w = depth.shape
        r = C.c_void_p(L.orc_peac_run(depth.ctypes.data, w, h, K[0], K[1], K[2], K[3], float(np.float32(scale))))
        n = L.orc_peac_num_planes(r)
        self.n_coarse = L.orc_peac_num_coarse(r)
        self.labels = np.zeros((h, w), np.int32)
        L.orc_peac_labels(r, self.labels.ctypes.data)
        self.planes = []
        self.membership = []
        for i in range(n):
            d8 = np.zeros(8)
            i2 = np.zeros(2, np.int32)
            L.orc_peac_plane(r, i, d8.ctypes.data, i2.ctypes.data)
            self.planes.append((d8, i2))
            buf = np.zeros(h * w, np.int32)
            m = L.orc_peac_membership(r, i, buf.ctypes.data, h * w)
            self.membership.append(buf[:m].copy())
        nb = (h // 10) * (w // 10)
        self.blk_d = np.zeros((nb, 17))
        self.blk_i = np.zeros((nb, 2), np.int32)
        L.orc_peac_blocks(r, self.blk_d.ctypes.data, self.blk_i.ctypes.data)
        self.coarse_blocks = np.zeros(nb, np.int32)
        L.orc_peac_coarse_blocks(r, self.coarse_blocks.ctypes.data)
        L.orc_peac_free(r)


class _PoseProblemC(C.Structure):
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("bf", C.c_float),
                ("n_points", C.c_int32), ("Xw", C.c_void_p), ("obs", C.c_void_p), ("inv_sigma2", C.c_void_p),
                ("n_lines", C.c_int32), ("line_Xw", C.c_void_p), ("line_obs", C.c_void_p),
                ("n_planes", C.c_int32), ("n_par", C.c_int32), ("n_ver", C.c_int32),
                ("plane_meas", C.c_void_p), ("plane_map", C.c_void_p), ("par_meas", C.c_void_p), ("par_map", C.c_void_p),
                ("ver_meas", C.c_void_p), ("ver_map", C.c_void_p),
                ("angle_info", C.c_double), ("dist_info", C.c_double), ("par_info", C.c_double), ("ver_info", C.c_double),
                ("plane_chi", C.c_double), ("vp_chi", C.c_double)]


def pose_problem_struct(p: dict, cls=_PoseProblemC):
    """Build the C struct (shared layout between the oracle and the product ABI) from a synth_pose problem dict.
    Keeps references to the arrays alive on the returned object."""
    s = cls()
    s._keep = p
    for k in ("fx", "fy", "cx", "cy", "bf", "angle_info", "dist_info", "par_info", "ver_info", "plane_chi", "vp_chi"):
        setattr(s, k, p[k])
    s.n_points, s.n_lines = len(p["Xw"]), len(p["line_Xw"])
    s.n_planes, s.n_par, s.n_ver = len(p["plane_meas"]), len(p["par_meas"]), len(p["ver_meas"])
    for k in ("Xw", "obs", "inv_sigma2", "line_Xw", "line_obs", "plane_meas", "plane_map", "par_meas", "par_map", "ver_meas", "ver_map"):
        setattr(s, k, p[k].ctypes.data if p[k].size else None)
    return s


def translation_optimization(p: dict):
    return pose_optimization(p, translation_only=True)


def pose_optimization(p: dict, translation_only: bool = False):
    """Oracle PoseOptimization / TranslationOptimization. Returns dict(Tcw float 4x4, Tcw_d, n_inliers, outlier flags, trace)."""
    L = lib()
    L.orc_pose_optimization.argtypes = [C.c_void_p] * 11
    L.orc_translation_optimization.argtypes = [C.c_void_p] * 11
    s = pose_problem_struct(p)
    T0 = np.ascontiguousarray(p["Tcw0"], np.float32)
    T = np.zeros((4, 4), np.float32)
    Td = np.zeros((4, 4))
    o = [np.zeros(max(n, 1), np.uint8) for n in (s.n_points, s.n_lines, s.n_planes, s.n_par, s.n_ver)]
    ti, td = np.zeros((4, 3), np.int32), np.zeros((4, 2))
    fn = L.orc_translation_optimization if translation_only else L.orc_pose_optimization
    n = fn(C.byref(s), T0.ctypes.data, T.ctypes.data, Td.ctypes.data, *[a.ctypes.data for a in o], ti.ctypes.data,
                                td.ctypes.data)
    return dict(Tcw=T, Tcw_d=Td, n_inliers=n, outlier_pt=o[0][:s.n_points], outlier_line=o[1][:s.n_lines], outlier_plane=o[2][:s.n_planes],
                outlier_par=o[3][:s.n_par], outlier_ver=o[4][:s.n_ver], trace_i=ti, trace_d=td)


class _FrameViewC(C.Structure):
    _fields_ = [("n", C.c_int32), ("keys_un", C.c_void_p), ("u_right", C.c_void_p), ("desc", C.c_void_p), ("Tcw", C.c_float * 16),
                ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("bf", C.c_float),
                ("min_x", C.c_float), ("max_x", C.c_float), ("min_y", C.c_float), ("max_y", C.c_float),
                ("n_levels", C.c_int32), ("scale_factors", C.c_void_p), ("log_scale_factor", C.c_float)]


class _MapPointsC(C.Structure):
    _fields_ = [("n", C.c_int32), ("pos", C.c_void_p), ("normal", C.c_void_p), ("max_distance", C.c_void_p), ("min_distance", C.c_void_p),
                ("desc", C.c_void_p), ("skip", C.c_void_p), ("has_obs", C.c_void_p)]


class _LastFrameC(C.Structure):
    _fields_ = [("n", C.c_int32), ("keys", C.c_void_p), ("map_point", C.c_void_p), ("outlier", C.c_void_p), ("Tcw", C.c_float * 16)]


def frame_view_struct(fv: dict, cls=_FrameViewC):
    s = cls()
    s._keep = fv
    s.n = fv["n"]
    for k in ("keys_un", "u_right", "desc", "scale_factors"):
        setattr(s, k, fv[k].ctypes.data)
    s.Tcw = (C.c_float * 16)(*np.asarray(fv["Tcw"], np.float32).ravel().tolist())
    for k in ("fx", "fy", "cx", "cy", "bf", "min_x", "max_x", "min_y", "max_y", "log_scale_factor"):
        setattr(s, k, fv[k])
    s.n_levels = fv["n_levels"]
    return s


def map_points_struct(m: dict, cls=_MapPointsC):
    s = cls()
    s._keep = m
    s.n = m["n"]
    for k in ("pos", "normal", "max_distance", "min_distance", "desc", "skip", "has_obs"):
        setattr(s, k, m[k].ctypes.data)
    return s


def last_frame_struct(lf: dict, cls=_LastFrameC):
    s = cls()
    s._keep = lf
    s.n = lf["n"]
    for k in ("keys", "map_point", "outlier"):
        setattr(s, k, lf[k].ctypes.data)
    s.Tcw = (C.c_float * 16)(*np.asarray(lf["Tcw"], np.float32).ravel().tolist())
    return s


def search_by_projection_map(fv: dict, m: dict, th: float, nnratio: float, matches0: np.ndarray):
    L = lib()
    L.orc_search_by_projection_map.argtypes = [C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
    matches = np.ascontiguousarray(matches0, np.int32).copy()
    in_view = np.zeros(max(m["n"], 1), np.uint8)
    n = L.orc_search_by_projection_map(C.byref(frame_view_struct(fv)), C.byref(map_points_struct(m)), th, nnratio, matches.ctypes.data,
                                       in_view.ctypes.data)
    return n, matches, in_view[:m["n"]]


def search_by_projection_last(fv: dict, lf: dict, m: dict, th: float, mono: bool, check_ori: bool, matches0: np.ndarray):
    L = lib()
    L.orc_search_by_projection_last.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_int, C.c_int, C.c_void_p]
    matches = np.ascontiguousarray(matches0, np.int32).copy()
    n = L.orc_search_by_projection_last(C.byref(frame_view_struct(fv)), C.byref(last_frame_struct(lf)), C.byref(map_points_struct(m)), th,
                                        int(mono), int(check_ori), matches.ctypes.data)
    return n, matches


def local_bundle_adjustment(p: dict) -> dict:
    """Oracle Optimizer::LocalBundleAdjustment on a planarslam_b200.synth_lba problem dict (same ctypes mirror as the ABI)."""
    from planarslam_b200 import lba as _lba
    L = lib()
    L.orc_local_bundle_adjustment.argtypes = [C.c_void_p, C.c_void_p]
    s = _lba.problem_struct(p)
    r, o = _lba.result_struct(s)
    rc = L.orc_local_bundle_adjustment(C.byref(s), C.byref(r))
    assert rc == 0
    return _lba.finish(r, o)


KEYLINE_DTYPE = np.dtype([("angle", "<f4"), ("class_id", "<i4"), ("octave", "<i4"), ("pt", "<f4", 2), ("response", "<f4"), ("size", "<f4"),
                          ("startPointX", "<f4"), ("startPointY", "<f4"), ("endPointX", "<f4"), ("endPointY", "<f4"),
                          ("sPointInOctaveX", "<f4"), ("sPointInOctaveY", "<f4"), ("ePointInOctaveX", "<f4"), ("ePointInOctaveY", "<f4"),
                          ("lineLength", "<f4"), ("numOfPixels", "<i4")])
assert KEYLINE_DTYPE.itemsize == 68


def lsd_detect(gray: np.ndarray, refine: int = 2, cap: int = 16384, rect_enum: int = 1):
    """Oracle cv::LineSegmentDetector::detect. Returns (segments float32 [n][4], width, prec, nfa float64 [n]).
    rect_enum: NFA pixel enumeration - 1 cv2 4.13's with the deterministic sincos (the CUDA path's default, oracle/lsd.cc rect_nfa),
    0 the published LSD iterator, 3 cv2 4.13's with libm axes (= cv2 bit for bit)."""
    L = lib()
    L.orc_lsd_detect_enum.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    g = np.ascontiguousarray(gray, np.uint8)
    segs, wpn = np.zeros((cap, 4), np.float32), np.zeros((cap, 3))
    n = L.orc_lsd_detect_enum(g.ctypes.data, g.shape[1], g.shape[0], g.strides[0], refine, rect_enum, segs.ctypes.data, wpn.ctypes.data, cap)
    assert n <= cap
    return segs[:n].copy(), wpn[:n, 0].copy(), wpn[:n, 1].copy(), wpn[:n, 2].copy()


def lsd_stages(gray: np.ndarray, refine: int = 2):
    """Intermediate products of the oracle detector (for the GPU stage-parity tests)."""
    L = lib()
    L.orc_lsd_stages.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 7
    g = np.ascontiguousarray(gray, np.uint8)
    h, w = g.shape
    sw, sh = int(round(w * 0.8)), int(round(h * 0.8))
    out = dict(blurred=np.zeros((h, w), np.uint8), scaled=np.zeros((sh, sw), np.uint8), modgrad=np.zeros((sh, sw)), angles=np.zeros((sh, sw)),
               order=np.zeros((sw - 1) * (sh - 1), np.int32), region_id=np.zeros((sh, sw), np.int32))
    dims = np.zeros(2, np.int32)
    n = L.orc_lsd_stages(g.ctypes.data, w, h, g.strides[0], refine, out["blurred"].ctypes.data, out["scaled"].ctypes.data, out["modgrad"].ctypes.data,
                         out["angles"].ctypes.data, out["order"].ctypes.data, out["region_id"].ctypes.data, dims.ctypes.data)
    assert (dims[0], dims[1]) == (sw, sh)
    out["n_segments"] = n
    return out


def extract_line_segments(gray: np.ndarray, max_lines: int = 40, rect_enum: int = 1):
    """Oracle LineSegment::ExtractLineSegment without LBD. Returns (KeyLine structured array, line functions [n][3])."""
    L = lib()
    L.orc_extract_line_segments_enum.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    g = np.ascontiguousarray(gray, np.uint8)
    cap = max(max_lines, 1)
    kl, lf = np.zeros(cap, KEYLINE_DTYPE), np.zeros((cap, 3))
    n = L.orc_extract_line_segments_enum(g.ctypes.data, g.shape[1], g.shape[0], g.strides[0], max_lines, rect_enum, kl.ctypes.data, lf.ctypes.data, cap)
    return kl[:n].copy(), lf[:n].copy()


def line_search_by_projection(frame: dict, map_lines: dict, th: float, nnratio: float):
    """Oracle LSDmatcher::SearchByProjection(Frame&, vector<MapLine*>&, th).  Same dict layout as planarslam_b200.matcher.LSDmatcher."""
    L = lib()
    L.orc_line_search_by_projection.argtypes = [C.c_int] + [C.c_void_p] * 6 + [C.c_int, C.c_int] + [C.c_void_p] * 6 + [C.c_float, C.c_float, C.c_void_p]
    f = {k: np.ascontiguousarray(v) for k, v in frame.items()}
    m = {k: np.ascontiguousarray(v) for k, v in map_lines.items()}
    nf, nm = len(f["angle"]), len(m["level"])
    assigned = np.full(max(nf, 1), -1, np.int32)
    n = L.orc_line_search_by_projection(nf, f["pt"].ctypes.data, f["angle"].ctypes.data, f["octave"].ctypes.data, f["desc"].ctypes.data,
                                        f["has_obs"].ctypes.data, f["scale_factors"].ctypes.data, len(f["scale_factors"]), nm, m["skip"].ctypes.data,
                                        m["level"].ctypes.data, m["view_cos"].ctypes.data, m["proj"].ctypes.data, m["desc"].ctypes.data,
                                        m["has_obs"].ctypes.data, th, nnratio, assigned.ctypes.data)
    return n, assigned[:nf]


def search_by_bow(kf: dict, frame: dict, nnratio: float = 0.7, check_orientation: bool = True):
    """Oracle ORBmatcher::SearchByBoW(KeyFrame*, Frame&, ...).  Same dict layout as planarslam_b200.matcher.search_by_bow."""
    L = lib()
    L.orc_search_by_bow.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_int, C.c_void_p]
    k = {a: np.ascontiguousarray(b) for a, b in kf.items()}
    f = {a: np.ascontiguousarray(b) for a, b in frame.items()}
    nf = len(f["angle"])
    match = np.full(max(nf, 1), -1, np.int32)
    n = L.orc_search_by_bow(len(k["angle"]), k["desc"].ctypes.data, k["angle"].ctypes.data, k["has_mp"].ctypes.data, len(k["node_id"]), k["node_id"].ctypes.data,
                            k["node_off"].ctypes.data, k["node_feat"].ctypes.data, nf, f["desc"].ctypes.data, f["angle"].ctypes.data, len(f["node_id"]),
                            f["node_id"].ctypes.data, f["node_off"].ctypes.data, f["node_feat"].ctypes.data, nnratio, 1 if check_orientation else 0,
                            match.ctypes.data)
    return n, match[:nf]


def bow_transform(voc: dict, features: np.ndarray, levelsup: int = 4):
    """Oracle DBoW2 TemplatedVocabulary::transform (TF_IDF, L1).  Returns dict(word_id, word_val, node_id, node_off, node_feat, feat_word, feat_node)."""
    L = lib()
    L.orc_bow_transform.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 6 + [C.c_int, C.c_int] + [C.c_void_p] * 8
    f = np.ascontiguousarray(features, np.uint8)
    n = len(f)
    o = dict(word_id=np.zeros(n, np.int32), word_val=np.zeros(n), node_id=np.zeros(n, np.int32), node_off=np.zeros(n + 1, np.int32),
             node_feat=np.zeros(n, np.int32), feat_word=np.zeros(n, np.int32), feat_node=np.zeros(n, np.int32))
    cnt = np.zeros(2, np.int32)
    L.orc_bow_transform(len(voc["word_id"]), voc["L"], voc["desc"].ctypes.data, voc["child_off"].ctypes.data, voc["child_id"].ctypes.data,
                        voc["word_id"].ctypes.data, voc["weight"].ctypes.data, f.ctypes.data, n, levelsup, o["word_id"].ctypes.data,
                        o["word_val"].ctypes.data, o["node_id"].ctypes.data, o["node_off"].ctypes.data, o["node_feat"].ctypes.data,
                        o["feat_word"].ctypes.data, o["feat_node"].ctypes.data, cnt.ctypes.data)
    nw, nn = int(cnt[0]), int(cnt[1])
    o["word_id"], o["word_val"] = o["word_id"][:nw], o["word_val"][:nw]
    o["node_id"], o["node_off"] = o["node_id"][:nn], o["node_off"][:nn + 1]
    o["node_feat"] = o["node_feat"][:o["node_off"][-1]] if nn else o["node_feat"][:0]
    return o


def bow_score_l1(a: dict, b: dict) -> float:
    L = lib()
    L.orc_bow_score_l1.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    L.orc_bow_score_l1.restype = C.c_double
    return float(L.orc_bow_score_l1(a["word_id"].ctypes.data, a["word_val"].ctypes.data, len(a["word_id"]), b["word_id"].ctypes.data,
                                    b["word_val"].ctypes.data, len(b["word_id"])))


def glibc_rand(seed: int, n: int) -> np.ndarray:
    """The first n values of rand() after srand(seed), from the oracle's restatement of glibc's TYPE_3 generator."""
    L = lib()
    L.orc_glibc_rand.argtypes = [C.c_uint32, C.c_int, C.c_void_p]
    out = np.zeros(n, np.int32)
    L.orc_glibc_rand(seed, n, out.ctypes.data)
    return out


def cv_svd(A: np.ndarray):
    """cv::SVD::compute (no FULL_UV) by OpenCV's Jacobi algorithm (oracle/cvsvd.h). Returns (w, u, vt)."""
    L = lib()
    A = np.ascontiguousarray(A)
    assert A.dtype in (np.float32, np.float64) and A.ndim == 2
    m, n = A.shape
    k = min(m, n)
    w, u, vt = np.zeros(k, A.dtype), np.zeros((m, k), A.dtype), np.zeros((k, n), A.dtype)
    fn = L.orc_cv_svd64 if A.dtype == np.float64 else L.orc_cv_svd32
    fn.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    fn(A.ctypes.data, m, n, w.ctypes.data, u.ctypes.data, vt.ctypes.data)
    return w, u, vt


def lines3d_frame(keylines: np.ndarray, depth: np.ndarray, cam, seed: int = 1, skip: int = 0):
    """Oracle Frame::isLineGood for one frame. keylines: KEYLINE_DTYPE[n]; depth float32 [h][w] metres; cam (fx, fy, cx, cy).
    Returns dict(valid, depth_line, lines3d [n][6], director [n][3], n_points, n_inliers, inliers u64, n_drawn)."""
    L = lib()
    L.orc_lines3d_frame.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint32, C.c_int] + [C.c_void_p] * 7
    kl = np.ascontiguousarray(keylines, KEYLINE_DTYPE)
    d = np.ascontiguousarray(depth, np.float32)
    n = len(kl)
    camv = np.asarray(cam, np.float32)
    o = dict(valid=np.zeros(n, np.uint8), depth_line=np.zeros(n, np.float32), lines3d=np.zeros((n, 6)), director=np.zeros((n, 3)),
             n_points=np.zeros(n, np.int32), n_inliers=np.zeros(n, np.int32), inliers=np.zeros(n, np.uint64))
    o["n_drawn"] = L.orc_lines3d_frame(kl.ctypes.data, n, d.ctypes.data, d.shape[1], d.shape[0], camv.ctypes.data, seed, skip, o["valid"].ctypes.data,
                                       o["depth_line"].ctypes.data, o["lines3d"].ctypes.data, o["director"].ctypes.data, o["n_points"].ctypes.data,
                                       o["n_inliers"].ctypes.data, o["inliers"].ctypes.data)
    return o


def track_manhattan_frame(R_last: np.ndarray, normals: np.ndarray, dirs: np.ndarray):
    """Oracle Tracking::TrackManhattanFrame. R_last 3x3 float32, normals [n][3] float32, dirs [m][3] float64.
    Returns dict(R, found, density, n_cone, n_selected, min_num, svd_applied, normal_mask, dir_mask)."""
    L = lib()
    L.orc_track_manhattan_frame.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    R = np.ascontiguousarray(R_last, np.float32).reshape(3, 3)
    nr = np.ascontiguousarray(normals, np.float32).reshape(-1, 3)
    dr = np.ascontiguousarray(dirs, np.float64).reshape(-1, 3)
    oi, of = np.zeros(11, np.int32), np.zeros(12, np.float32)
    nm, dm = np.zeros(max(len(nr), 1), np.uint8), np.zeros(max(len(dr), 1), np.uint8)
    L.orc_track_manhattan_frame(R.ctypes.data, nr.ctypes.data, len(nr), dr.ctypes.data, len(dr), oi.ctypes.data, of.ctypes.data, nm.ctypes.data, dm.ctypes.data)
    return dict(R=of[:9].reshape(3, 3).copy(), density=of[9:].copy(), found=oi[:3].copy(), n_cone=oi[3:6].copy(), n_selected=oi[6:9].copy(), min_num=int(oi[9]),
                svd_applied=int(oi[10]), normal_mask=nm[:len(nr)].copy(), dir_mask=dm[:len(dr)].copy())


def lines_in_frustum(frame: dict, pos, normal, max_distance, min_distance, cos_limit: float = 0.6):
    """Oracle Frame::isInFrustum(MapLine*, cosLimit) for n map lines. frame: dict(Tcw 4x4, fx, fy, cx, cy, min_x, max_x, min_y, max_y, log_scale_factor).
    Returns dict(in_view, proj [n][4], level, view_cos)."""
    L = lib()
    L.orc_lines_in_frustum.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float] + [C.c_void_p] * 4
    fv = np.concatenate([np.asarray(frame["Tcw"], np.float32).ravel(), np.array([frame[k] for k in ("fx", "fy", "cx", "cy", "min_x", "max_x", "min_y", "max_y",
                                                                                                      "log_scale_factor")], np.float32)])
    P, Nn = np.ascontiguousarray(pos, np.float64).reshape(-1, 6), np.ascontiguousarray(normal, np.float64).reshape(-1, 3)
    mx, mn = np.ascontiguousarray(max_distance, np.float32), np.ascontiguousarray(min_distance, np.float32)
    n = len(P)
    o = dict(in_view=np.zeros(n, np.uint8), proj=np.zeros((n, 4), np.float32), level=np.zeros(n, np.int32), view_cos=np.zeros(n, np.float32))
    L.orc_lines_in_frustum(fv.ctypes.data, n, P.ctypes.data, Nn.ctypes.data, mx.ctypes.data, mn.ctypes.data, cos_limit, o["in_view"].ctypes.data, o["proj"].ctypes.data,
                           o["level"].ctypes.data, o["view_cos"].ctypes.data)
    return o


def compute_stereo_from_rgbd(keys_xy, keys_un_xy, depth, bf: float):
    """Oracle Frame::ComputeStereoFromRGBD. keys_xy / keys_un_xy [n][2] float32, depth float32 [h][w]. Returns (mvuRight, mvDepth)."""
    L = lib()
    L.orc_compute_stereo_from_rgbd.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_void_p]
    k, ku = np.ascontiguousarray(keys_xy, np.float32), np.ascontiguousarray(keys_un_xy, np.float32)
    d = np.ascontiguousarray(depth, np.float32)
    n = len(k)
    ur, dz = np.zeros(n, np.float32), np.zeros(n, np.float32)
    L.orc_compute_stereo_from_rgbd(n, k.ctypes.data, ku.ctypes.data, d.ctypes.data, d.shape[1], bf, ur.ctypes.data, dz.ctypes.data)
    return ur, dz


def lbd_compute(gray: np.ndarray, keylines: np.ndarray):
    """Oracle BinaryDescriptor::compute (oracle/lbd.cc; descriptor logic parity-unpinned, see oracle/lbd.h).  Returns (lbd float32 [n][72], desc uint8 [n][32])."""
    L = lib()
    L.orc_lbd_compute.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.orc_lbd_compute.restype = None
    g = np.ascontiguousarray(gray, np.uint8)
    kl = np.ascontiguousarray(keylines, KEYLINE_DTYPE)
    n = len(kl)
    f, d = np.zeros((max(n, 1), 72), np.float32), np.zeros((max(n, 1), 32), np.uint8)
    L.orc_lbd_compute(g.ctypes.data, g.shape[1], g.shape[0], g.strides[0], kl.ctypes.data, n, f.ctypes.data, d.ctypes.data)
    return f[:n], d[:n]


def lbd_prims(gray: np.ndarray):
    """(GaussianBlur 5x5 s=1, Sobel dx, Sobel dy of the blurred image) as the LBD oracle computes them."""
    L = lib()
    L.orc_gaussian_blur_5x5_s1.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.orc_sobel3_s16.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    g = np.ascontiguousarray(gray, np.uint8)
    h, w = g.shape
    b, dx, dy = np.zeros((h, w), np.uint8), np.zeros((h, w), np.int16), np.zeros((h, w), np.int16)
    L.orc_gaussian_blur_5x5_s1(g.ctypes.data, w, h, g.strides[0], b.ctypes.data)
    L.orc_sobel3_s16(b.ctypes.data, w, h, dx.ctypes.data, dy.ctypes.data)
    return b, dx, dy


def planes_post(depth: np.ndarray, K=(535.4, 539.2, 320.1, 247.6), scale=np.float32(1.0 / 5000.0), dist_th: float = 0.05):
    """Oracle Frame::ComputePlanes post-processing (PEAC -> VoxelGrid 0.1 -> MaxPointDistanceFromPlane check -> RANSAC refit; oracle/planepost.cc, parity
    unpinned).  Returns a list of dict(src, coef float32 [4], points float32 [n][3], n_inliers, n_iterations)."""
    L = lib()
    depth = np.ascontiguousarray(depth, np.uint16)
    h, w = depth.shape
    r = C.c_void_p(L.orc_peac_run(depth.ctypes.data, w, h, K[0], K[1], K[2], K[3], float(np.float32(scale))))
    L.orc_planes_post.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int] + [C.c_float] * 5 + [C.c_double] + [C.c_void_p] * 4 + [C.c_int, C.c_void_p]
    cap = 128
    src, coef, npts, stats = np.zeros(cap, np.int32), np.zeros((cap, 4), np.float32), np.zeros(cap, np.int32), np.zeros((cap, 2), np.int32)
    pts = np.zeros((200000, 3), np.float32)
    n = L.orc_planes_post(r, depth.ctypes.data, w, h, K[0], K[1], K[2], K[3], float(np.float32(scale)), dist_th, src.ctypes.data, coef.ctypes.data, npts.ctypes.data,
                          pts.ctypes.data, len(pts), stats.ctypes.data)
    L.orc_peac_free(r)
    out, o = [], 0
    for i in range(n):
        out.append(dict(src=int(src[i]), coef=coef[i].copy(), points=pts[o:o + npts[i]].copy(), n_inliers=int(stats[i, 0]), n_iterations=int(stats[i, 1])))
        o += int(npts[i])
    return out


def planes_post_records(depth: np.ndarray, normal_center: np.ndarray, members: list, K, scale, dist_th: float = 0.05):
    """planes_post on caller-made plane records instead of a PEAC run: normal_center float64 [n][6] (PEAC normal, centre), members = one array of pixel
    indices per plane.  Same return layout as planes_post."""
    L = lib()
    depth = np.ascontiguousarray(depth, np.uint16)
    h, w = depth.shape
    L.orc_planes_post_records.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_float] * 5 + [C.c_double, C.c_int] + [C.c_void_p] * 7 + [C.c_int, C.c_void_p]
    nc = np.ascontiguousarray(normal_center, np.float64).reshape(-1, 6)
    off = np.concatenate([[0], np.cumsum([len(m) for m in members])]).astype(np.int32)
    idx = np.ascontiguousarray(np.concatenate(members) if members else np.zeros(0), np.int32)
    cap = max(len(nc), 1)
    src, coef, npts, stats = np.zeros(cap, np.int32), np.zeros((cap, 4), np.float32), np.zeros(cap, np.int32), np.zeros((cap, 2), np.int32)
    pts = np.zeros((200000, 3), np.float32)
    n = L.orc_planes_post_records(depth.ctypes.data, w, h, K[0], K[1], K[2], K[3], float(np.float32(scale)), dist_th, len(nc), nc.ctypes.data, off.ctypes.data,
                                  idx.ctypes.data, src.ctypes.data, coef.ctypes.data, npts.ctypes.data, pts.ctypes.data, len(pts), stats.ctypes.data)
    out, o = [], 0
    for i in range(n):
        out.append(dict(src=int(src[i]), coef=coef[i].copy(), points=pts[o:o + npts[i]].copy(), n_inliers=int(stats[i, 0]), n_iterations=int(stats[i, 1])))
        o += int(npts[i])
    return out


def surface_normals(depth: np.ndarray, K=(535.4, 539.2, 320.1, 247.6), scale=np.float32(1.0 / 5000.0)):
    """Oracle vSurfaceNormal of Frame::ComputePlanes (IntegralImageNormalEstimation AVERAGE_3D_GRADIENT restated; parity unpinned): float32 [n][8] =
    normal xyz (NaN at the borders / depth edges), camera position xyz, frame position xy."""
    L = lib()
    L.orc_surface_normals.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_float] * 5 + [C.c_void_p, C.c_int]
    depth = np.ascontiguousarray(depth, np.uint16)
    h, w = depth.shape
    cap = ((h + 2) // 3) * ((w + 2) // 3)
    out = np.zeros((cap, 8), np.float32)
    n = L.orc_surface_normals(depth.ctypes.data, w, h, K[0], K[1], K[2], K[3], float(np.float32(scale)), out.ctypes.data, cap)
    return out[:n].copy()


def _db_args(db):
    d = {k: np.ascontiguousarray(v) for k, v in db.items()}
    n_kf = len(d["off"]) - 1
    covis = d.get("covis")
    return d, n_kf, (covis.ctypes.data if covis is not None else None), (covis.shape[1] if covis is not None else 0)


def detect_loop_candidates(db: dict, min_score: float, sentinel: float = -1.0):
    """Oracle KeyFrameDatabase::DetectLoopCandidates.  db: planarslam_b200.synth_lines.make_bow_database layout.  Returns (candidates, common_words, score);
    score[k] == sentinel where the reference does not evaluate it."""
    L = lib()
    L.orc_detect_loop_candidates.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_void_p, C.c_float] + [C.c_void_p] * 3
    d, n_kf, covis, stride = _db_args(db)
    cand, words, score = np.zeros(max(n_kf, 1), np.int32), np.zeros(max(n_kf, 1), np.int32), np.full(max(n_kf, 1), sentinel, np.float32)
    n = L.orc_detect_loop_candidates(d["q_word"].ctypes.data, d["q_val"].ctypes.data, len(d["q_word"]), n_kf, d["off"].ctypes.data, d["word"].ctypes.data,
                                     d["val"].ctypes.data, covis, stride, d["connected"].ctypes.data if "connected" in d else None, min_score,
                                     cand.ctypes.data, words.ctypes.data, score.ctypes.data)
    return cand[:n].copy(), words[:n_kf], score[:n_kf]


def detect_relocalization_candidates(db: dict, reloc_score: np.ndarray):
    """Oracle KeyFrameDatabase::DetectRelocalizationCandidates.  reloc_score = KeyFrame::mRelocScore before the call.  Returns (candidates, common_words, mRelocScore after)."""
    L = lib()
    L.orc_detect_relocalization_candidates.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 4 + [C.c_int] + [C.c_void_p] * 3
    d, n_kf, covis, stride = _db_args(db)
    cand, words, score = np.zeros(max(n_kf, 1), np.int32), np.zeros(max(n_kf, 1), np.int32), np.ascontiguousarray(reloc_score, np.float32).copy()
    n = L.orc_detect_relocalization_candidates(d["q_word"].ctypes.data, d["q_val"].ctypes.data, len(d["q_word"]), n_kf, d["off"].ctypes.data, d["word"].ctypes.data,
                                               d["val"].ctypes.data, covis, stride, score.ctypes.data, cand.ctypes.data, words.ctypes.data)
    return cand[:n].copy(), words[:n_kf], score


def _bow_kf_call(fn, kf1, kf2, nnratio, check_orientation):
    fn.argtypes = ([C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p] * 2) + [C.c_float, C.c_int, C.c_void_p]
    a = {k: np.ascontiguousarray(v) for k, v in kf1.items()}
    b = {k: np.ascontiguousarray(v) for k, v in kf2.items()}
    n1 = len(a["angle"])
    match = np.full(max(n1, 1), -1, np.int32)
    side = lambda s: (len(s["angle"]), s["desc"].ctypes.data, s["angle"].ctypes.data, s["has_mp"].ctypes.data, len(s["node_id"]), s["node_id"].ctypes.data,
                      s["node_off"].ctypes.data, s["node_feat"].ctypes.data)
    n = fn(*side(a), *side(b), nnratio, 1 if check_orientation else 0, match.ctypes.data)
    return n, match[:n1]


def search_by_bow_kf(kf1: dict, kf2: dict, nnratio: float = 0.75, check_orientation: bool = True):
    """Oracle ORBmatcher::SearchByBoW(KeyFrame*, KeyFrame*, vector<MapPoint*>&).  Returns (nmatches, match12 [n1]: feature of key frame 2 or -1)."""
    return _bow_kf_call(lib().orc_search_by_bow_kf, kf1, kf2, nnratio, check_orientation)


def map_plane_update(clouds):
    """Oracle MapPlane::UpdateCoefficientsAndPoints (oracle/planepost.cc map_plane_update, parity unpinned): clouds = [(points float32 [k][3], T float64 [4][4])].
    Returns the voxel centroids float32 [n][3]."""
    L = lib()
    L.orc_map_plane_update.argtypes = [C.c_int] + [C.c_void_p] * 4 + [C.c_int]
    off, pts, Ts = [0], [], []
    for p, T in clouds:
        p = np.ascontiguousarray(p, np.float32).reshape(-1, 3)
        pts.append(p); Ts.append(np.ascontiguousarray(T, np.float64).reshape(16)); off.append(off[-1] + len(p))
    off = np.asarray(off, np.int32)
    P = np.ascontiguousarray(np.concatenate(pts) if pts else np.zeros((0, 3), np.float32))
    T = np.ascontiguousarray(np.stack(Ts) if Ts else np.zeros((0, 16)))
    out = np.zeros((max(len(P), 1), 3), np.float32)
    n = L.orc_map_plane_update(len(clouds), off.ctypes.data, P.ctypes.data, T.ctypes.data, out.ctypes.data, len(out))
    return out[:n].copy()
