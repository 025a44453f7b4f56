"""Host-side mirror of the reference's ORBextractor (include/ORBextractor.h:47-116) on top of the C ABI.

Same constructor arguments, getters and call shape as the reference class; the work happens in
libpslam_b200.so (CUDA, sm_90a).  Images are numpy uint8 arrays, keypoints come back as a structured
array layout-compatible with cv::KeyPoint (28 bytes), descriptors as an N x 32 uint8 array.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import Context, KEYPOINT_DTYPE, E_CAPACITY


class ORBextractor:
    def __init__(self, nfeatures: int = 1000, scaleFactor: float = 1.2, nlevels: int = 8, iniThFAST: int = 20,
                 minThFAST: int = 7, device: int = 0, max_batch: int = 1):
        self.nfeatures, self.scaleFactor, self.nlevels = int(nfeatures), float(scaleFactor), int(nlevels)
        self.iniThFAST, self.minThFAST = int(iniThFAST), int(minThFAST)
        self.device, self.max_batch = device, max_batch
        self._ctx: Context | None = None
        self._shape = None

    # -- context management: the reference object is size-agnostic, a GPU context is not --------------
    def _context(self, h: int, w: int, batch: int) -> Context:
        if self._ctx is None or self._shape != (h, w) or batch > self._ctx.cfg.max_batch:
            if self._ctx is not None:
                self._ctx.close()
            self._ctx = Context(w, h, max(batch, self.max_batch), self.device, nfeatures=self.nfeatures,
                                scale_factor=self.scaleFactor, nlevels=self.nlevels, ini_th_fast=self.iniThFAST,
                                min_th_fast=self.minThFAST)
            self._shape = (h, w)
        return self._ctx

    def context(self, h: int, w: int, batch: int = 1) -> Context:
        return self._context(h, w, batch)

    # -- operator()(image, mask, keypoints, descriptors), include/ORBextractor.h:59-61 ----------------
    def __call__(self, image: np.ndarray, mask=None):
        if image is None or image.size == 0:           # reference: silent return on empty input (:1046)
            return np.zeros(0, KEYPOINT_DTYPE), np.zeros((0, 32), np.uint8)
        k, d = self.extract_batch(image[None])
        return k[0], d[0]

    def extract_batch(self, images: np.ndarray):
        """images: [B, H, W] uint8 -> (list of keypoint arrays, list of descriptor arrays)."""
        if images.dtype != np.uint8 or images.ndim != 3:
            raise TypeError("images must be a [B, H, W] uint8 array (CV_8UC1, reference assert :1050)")
        images = np.ascontiguousarray(images)
        B, H, W = images.shape
        ctx = self._context(H, W, B)
        cap = ctx.L.pslam_orb_max_keypoints(ctx.h)
        kps = np.zeros((B, cap), KEYPOINT_DTYPE)
        desc = np.zeros((B, cap, 32), np.uint8)
        n = np.zeros(B, np.int32)
        ctx.check(ctx.L.pslam_orb_extract_batch(ctx.h, images.ctypes.data, B, kps.ctypes.data, desc.ctypes.data, cap,
                                                n.ctypes.data))
        return [kps[i, :n[i]].copy() for i in range(B)], [desc[i, :n[i]].copy() for i in range(B)]

    # -- getters, include/ORBextractor.h:63-83 ---------------------------------------------------------
    def _tables(self):
        ctx = self._ctx or Context(640, 480, 1, self.device, nfeatures=self.nfeatures, scale_factor=self.scaleFactor,
                                   nlevels=self.nlevels, ini_th_fast=self.iniThFAST, min_th_fast=self.minThFAST)
        arrs = [np.zeros(self.nlevels, np.float32) for _ in range(4)] + [np.zeros(self.nlevels, np.int32)]
        fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        ctx.check(ctx.L.pslam_orb_get_scale_tables(ctx.h, *[a.ctypes.data_as(fp) for a in arrs[:4]], arrs[4].ctypes.data_as(ip)))
        return arrs

    def GetLevels(self): return self.nlevels
    def GetScaleFactor(self): return self.scaleFactor
    def GetScaleFactors(self): return self._tables()[0]
    def GetInverseScaleFactors(self): return self._tables()[1]
    def GetScaleSigmaSquares(self): return self._tables()[2]
    def GetInverseScaleSigmaSquares(self): return self._tables()[3]
    def GetFeaturesPerLevel(self): return self._tables()[4]

    # -- stage outputs for parity tests (mvImagePyramid is public in the reference, :85) -----------------
    def debug_level(self, frame: int, level: int, blurred: bool = False) -> np.ndarray:
        ctx = self._ctx
        w, h = C.c_int32(), C.c_int32()
        ctx.check(ctx.L.pslam_orb_debug_level_size(ctx.h, level, C.byref(w), C.byref(h)))
        out = np.zeros((h.value, w.value), np.uint8)
        fn = ctx.L.pslam_orb_debug_level_blurred if blurred else ctx.L.pslam_orb_debug_level_pixels
        ctx.check(fn(ctx.h, frame, level, out.ctypes.data))
        return out

    def debug_candidates(self, frame: int, level: int) -> np.ndarray:
        ctx = self._ctx
        cap = 200000
        buf = np.zeros((cap, 3), np.int32)
        n = C.c_int32()
        ctx.check(ctx.L.pslam_orb_debug_level_candidates(ctx.h, frame, level, buf.ctypes.data, cap, C.byref(n)))
        return buf[:n.value].copy()
