"""ctypes binding of libpslam_b200.so (the C ABI in include/pslam_abi.h).

There is deliberately no fallback: if the CUDA library is missing or no sm_90 GPU is present the
import / context creation fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpslam_b200.so")

KEYPOINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                           ("octave", "<i4"), ("class_id", "<i4")])
assert KEYPOINT_DTYPE.itemsize == 28

PLANE_DTYPE = np.dtype([("normal", "<f8", 3), ("center", "<f8", 3), ("mse", "<f8"), ("curvature", "<f8"), ("N", "<i4"), ("rid", "<i4")])
assert PLANE_DTYPE.itemsize == 72

PSLAM_OK, E_INVALID, E_NO_DEVICE, E_CUDA, E_CAPACITY, E_NCCL = 0, -1, -2, -3, -4, -5
# PSLAM_FRAME_CAP_*: the per-frame status bits of pslam_frame_construct_batch_dev
FRAME_CAP_ORB, FRAME_CAP_PEAC, FRAME_CAP_LINES, FRAME_CAP_PLANE_PTS = 1, 2, 4, 8


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("max_batch", C.c_int32),
                ("nfeatures", C.c_int32), ("scale_factor", C.c_float), ("nlevels", C.c_int32),
                ("ini_th_fast", C.c_int32), ("min_th_fast", C.c_int32),
                ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("depth_scale", C.c_float)]


class PoseProblem(C.Structure):
    """pslam_pose_problem (include/pslam_abi.h)."""
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("bf", C.c_float),
                ("n_points", C.c_int32), ("Xw", C.c_void_p), ("obs", C.c_void_p), ("inv_sigma2", C.c_void_p),
                ("n_lines", C.c_int32), ("line_Xw", C.c_void_p), ("line_obs", C.c_void_p),
                ("n_planes", C.c_int32), ("n_par", C.c_int32), ("n_ver", C.c_int32),
                ("plane_meas", C.c_void_p), ("plane_map", C.c_void_p), ("par_meas", C.c_void_p), ("par_map", C.c_void_p),
                ("ver_meas", C.c_void_p), ("ver_map", C.c_void_p),
                ("angle_info", C.c_double), ("dist_info", C.c_double), ("par_info", C.c_double), ("ver_info", C.c_double),
                ("plane_chi", C.c_double), ("vp_chi", C.c_double)]


class FrameView(C.Structure):
    _fields_ = [("n", C.c_int32), ("keys_un", C.c_void_p), ("u_right", C.c_void_p), ("desc", C.c_void_p), ("Tcw", C.c_float * 16),
                ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("bf", C.c_float),
                ("min_x", C.c_float), ("max_x", C.c_float), ("min_y", C.c_float), ("max_y", C.c_float),
                ("n_levels", C.c_int32), ("scale_factors", C.c_void_p), ("log_scale_factor", C.c_float)]


class MapPoints(C.Structure):
    _fields_ = [("n", C.c_int32), ("pos", C.c_void_p), ("normal", C.c_void_p), ("max_distance", C.c_void_p), ("min_distance", C.c_void_p),
                ("desc", C.c_void_p), ("skip", C.c_void_p), ("has_obs", C.c_void_p)]


class LastFrame(C.Structure):
    _fields_ = [("n", C.c_int32), ("keys", C.c_void_p), ("map_point", C.c_void_p), ("outlier", C.c_void_p), ("Tcw", C.c_float * 16)]


class PslamError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"pslam error {code}: {msg}")
        self.code = code


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, i32, f32p, i32p, u8p = C.c_void_p, C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_int32), C.c_void_p
    L.pslam_default_config.argtypes = [C.POINTER(Config), i32, i32, i32]; L.pslam_default_config.restype = None
    L.pslam_create.argtypes = [C.POINTER(Config), C.POINTER(vp)]
    L.pslam_destroy.argtypes = [vp]; L.pslam_destroy.restype = None
    L.pslam_last_error.argtypes = [vp]; L.pslam_last_error.restype = C.c_char_p
    L.pslam_set_stream.argtypes = [vp, vp]
    L.pslam_synchronize.argtypes = [vp]
    L.pslam_launch_count.argtypes = [vp]; L.pslam_launch_count.restype = C.c_int64
    L.pslam_profile_enable.argtypes = [vp, i32]
    L.pslam_profile_report.argtypes = [vp, C.c_char_p, i32]
    L.pslam_orb_get_scale_tables.argtypes = [vp, f32p, f32p, f32p, f32p, i32p]
    L.pslam_orb_max_keypoints.argtypes = [vp]
    L.pslam_orb_extract.argtypes = [vp, u8p, i32, vp, vp, i32, i32p]
    L.pslam_orb_extract_batch.argtypes = [vp, u8p, i32, vp, vp, i32, vp]
    L.pslam_orb_extract_batch_dev.argtypes = [vp, vp, i32, vp, vp, i32, vp]
    L.pslam_orb_debug_level_size.argtypes = [vp, i32, i32p, i32p]
    L.pslam_orb_debug_level_pixels.argtypes = [vp, i32, i32, vp]
    L.pslam_orb_debug_level_blurred.argtypes = [vp, i32, i32, vp]
    L.pslam_orb_debug_level_candidates.argtypes = [vp, i32, i32, vp, i32, i32p]
    L.pslam_peac_max_planes.argtypes = [vp]
    L.pslam_peac_num_blocks.argtypes = [vp]
    L.pslam_peac_wave_frames.argtypes = [vp]
    L.pslam_peac_run_batch.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp]
    L.pslam_peac_run_batch_dev.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp]
    L.pslam_peac_debug_blocks.argtypes = [vp, i32, vp, vp, vp, vp]
    L.pslam_peac_debug_coarse.argtypes = [vp, i32, vp, i32p]
    L.pslam_hamming_knn2.argtypes = [vp, vp, i32, vp, i32, vp, vp, vp, i32p]
    L.pslam_hamming_knn2_batch_dev.argtypes = [vp, vp, vp, i32, vp, vp, i32, i32, vp, vp, vp, vp]
    L.pslam_plane_match.argtypes = [vp, vp, i32, vp, i32, vp, vp, vp, vp, C.c_float, C.c_float, C.c_float, C.c_float, vp, vp, vp]
    L.pslam_search_by_projection_map.argtypes = [vp, vp, vp, C.c_float, C.c_float, vp, vp]
    L.pslam_search_by_projection_last.argtypes = [vp, vp, vp, vp, C.c_float, i32, i32, vp]
    L.pslam_pose_optimization.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    L.pslam_pose_optimization_batch.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp, vp, vp]
    L.pslam_pose_pack.argtypes = [vp, vp, i32, vp]
    L.pslam_translation_pack.argtypes = [vp, vp, i32, vp]
    L.pslam_translation_optimization.argtypes = [vp, vp, vp, vp, vp, vp]
    L.pslam_translation_optimization_batch.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp]
    L.pslam_pose_run_packed.argtypes = [vp]
    L.pslam_pose_fetch.argtypes = [vp] + [vp] * 10
    L.pslam_local_bundle_adjustment.argtypes = [vp, vp, vp]
    L.pslam_local_bundle_adjustment_batch.argtypes = [vp, vp, i32, vp]
    L.pslam_lba_pack.argtypes = [vp, vp, i32]
    L.pslam_lba_run_packed.argtypes = [vp]
    L.pslam_lba_fetch.argtypes = [vp, vp]
    L.pslam_lsd_max_segments.argtypes = [vp]
    L.pslam_lsd_set_rect_enumeration.argtypes = [vp, i32]
    L.pslam_lsd_detect_batch.argtypes = [vp, vp, i32, i32, vp, vp, i32, vp]
    L.pslam_lines_extract_batch.argtypes = [vp, vp, i32, i32, vp, vp, vp]
    L.pslam_lines_extract_batch_dev.argtypes = [vp, vp, i32, i32, vp, vp, vp]
    L.pslam_lsd_debug_stage.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp]
    L.pslam_lines3d_batch.argtypes = [vp, vp, vp, i32, vp, i32, C.c_float, vp, vp, vp, vp, vp]
    L.pslam_lines3d_batch_dev.argtypes = [vp, vp, vp, i32, vp, i32, C.c_float, vp, vp, vp, vp, vp]
    L.pslam_track_manhattan_batch.argtypes = [vp, vp, vp, vp, i32, vp, vp, i32, i32, vp, vp, vp]
    L.pslam_track_manhattan_batch_dev.argtypes = [vp, vp, vp, vp, i32, vp, vp, i32, i32, vp, vp, vp]
    L.pslam_lines_in_frustum.argtypes = [vp, vp, i32, vp, vp, vp, vp, C.c_float, vp, vp, vp, vp]
    L.pslam_compute_stereo_from_rgbd_batch.argtypes = [vp, vp, vp, vp, i32, vp, i32, C.c_float, C.c_float, vp, vp]
    L.pslam_compute_stereo_from_rgbd_batch_dev.argtypes = [vp, vp, vp, vp, i32, vp, i32, C.c_float, C.c_float, vp, vp]
    L.pslam_gray_from_color_batch_dev.argtypes = [vp, vp, i32, i32, i32, vp]
    L.pslam_frame_construct_batch_dev.argtypes = [vp, vp, vp, i32, C.c_float, C.c_float, C.c_float, i32, C.c_uint32, vp, vp]
    L.pslam_bow_transform.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp]
    L.pslam_bow_set_vocabulary.argtypes = [vp, i32, i32, vp, vp, vp, vp, vp]
    L.pslam_bow_transform_batch.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp]
    L.pslam_bow_transform_batch_dev.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp]
    L.pslam_search_by_bow.argtypes = [vp, i32, vp, vp, vp, i32, vp, vp, vp, i32, vp, vp, i32, vp, vp, vp, C.c_float, i32, vp]
    L.pslam_line_search_by_projection.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, C.c_float, C.c_float, vp]
    _lib = L
    return L


class Context:
    """Owns one pslam_ctx (one GPU, one stream)."""

    def __init__(self, width: int, height: int, max_batch: int = 1, device: int = 0, **overrides):
        L = lib()
        cfg = Config()
        L.pslam_default_config(C.byref(cfg), width, height, max_batch)
        cfg.device = device
        for k, v in overrides.items():
            if not hasattr(cfg, k):
                raise TypeError(f"unknown config field {k}")
            setattr(cfg, k, v)
        self.cfg = cfg
        h = C.c_void_p()
        rc = L.pslam_create(C.byref(cfg), C.byref(h))
        if rc != PSLAM_OK:
            raise PslamError(rc, "pslam_create failed (no sm_90 GPU, or invalid configuration; see stderr)")
        self.h = h
        self.L = L

    def check(self, rc: int, allow_capacity: bool = False) -> int:
        if rc == PSLAM_OK or (allow_capacity and rc == E_CAPACITY):
            return rc
        raise PslamError(rc, self.L.pslam_last_error(self.h).decode())

    def close(self):
        if getattr(self, "h", None):
            self.L.pslam_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream_ptr: int | None):
        self.check(self.L.pslam_set_stream(self.h, C.c_void_p(cuda_stream_ptr or 0)))

    def synchronize(self):
        self.check(self.L.pslam_synchronize(self.h))

    def profile(self, on: bool):
        self.check(self.L.pslam_profile_enable(self.h, 1 if on else 0))

    def profile_report(self) -> dict:
        """{kernel name: (launches, total_ms)} since profile(True)."""
        buf = C.create_string_buffer(1 << 16)
        self.check(self.L.pslam_profile_report(self.h, buf, len(buf)))
        out = {}
        for line in buf.value.decode().splitlines():
            name, n, ms = line.split()
            out[name] = (int(n), float(ms))
        return out

    @property
    def launch_count(self) -> int:
        return int(self.L.pslam_launch_count(self.h))
