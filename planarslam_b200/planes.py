"""Host-side mirror of the reference's PlaneDetection (include/PlaneExtractor.h:36-56) on top of the C ABI.

    pd = PlaneDetection()
    pd.readDepthImage(depth_u16, K, kScaleFactor)      # src/PlaneExtractor.cpp:26-57
    pd.runPlaneDetection(H, W)                         # src/PlaneExtractor.cpp:59-65
    pd.plane_num_, pd.plane_vertices_, pd.extractedPlanes, pd.membershipImg

The organised cloud (`cloud.vertices` in the reference) is not materialised; `vertex(i)` recomputes a point in
double exactly like readDepthImage does.
"""
from __future__ import annotations

import numpy as np

from ._lib import Context, PLANE_DTYPE


class PlaneDetection:
    def __init__(self, device: int = 0, max_batch: int = 1, **context_overrides):
        """context_overrides: Context settings other than the camera, e.g. nlevels - the context also holds the ORB pyramid geometry, and every pyramid
        level must be at least 68 pixels on a side, so frames smaller than 640 x 480 need fewer than the default 8 levels."""
        self.device, self.max_batch = device, max_batch
        self._overrides = context_overrides
        self._ctx: Context | None = None
        self._key = None
        self._depth = None
        self.plane_num_ = 0
        self.plane_vertices_: list[np.ndarray] = []
        self.extractedPlanes = np.zeros(0, PLANE_DTYPE)
        self.membershipImg = None

    def _context(self, h, w, K, scale, batch) -> Context:
        key = (h, w, tuple(np.float32(K).ravel().tolist()), float(np.float32(scale)))
        if self._ctx is None or self._key != key or batch > self._ctx.cfg.max_batch:
            if self._ctx is not None:
                self._ctx.close()
            K = np.asarray(K, np.float32)
            self._ctx = Context(w, h, max(batch, self.max_batch), self.device, fx=float(K[0, 0]), fy=float(K[1, 1]), cx=float(K[0, 2]),
                                cy=float(K[1, 2]), depth_scale=float(np.float32(scale)), **self._overrides)
            self._key = key
        return self._ctx

    # bool readDepthImage(cv::Mat depthImg, cv::Mat& K, float kScaleFactor)
    def readDepthImage(self, depthImg: np.ndarray, K: np.ndarray, kScaleFactor: float) -> bool:
        if depthImg is None or depthImg.size == 0 or depthImg.dtype != np.uint16:
            print("WARNING: cannot read depth image. No such a file, or the image format is not 16UC1")   # :34-38
            return False
        self._depth = np.ascontiguousarray(depthImg)
        self._K = np.asarray(K, np.float32)
        self._scale = np.float32(kScaleFactor)
        return True

    # void runPlaneDetection(int kDepthHeight, int kDepthWidth)
    def runPlaneDetection(self, kDepthHeight: int | None = None, kDepthWidth: int | None = None):
        res = self.run_batch(self._depth[None], self._K, self._scale)[0]
        self.membershipImg, self.extractedPlanes, self.plane_vertices_ = res
        self.plane_num_ = len(self.plane_vertices_)

    def run_batch(self, depth: np.ndarray, K, scale):
        """depth [B,H,W] uint16 -> list of (labels int32 [H,W], planes structured array, [pixel index arrays])."""
        depth = np.ascontiguousarray(depth)
        B, H, W = depth.shape
        ctx = self._context(H, W, K, scale, B)
        maxp = ctx.L.pslam_peac_max_planes(ctx.h)
        labels = np.zeros((B, H, W), np.int32)
        planes = np.zeros((B, maxp), PLANE_DTYPE)
        npl = np.zeros(B, np.int32)
        midx = np.zeros((B, H * W), np.int32)
        moff = np.zeros((B, maxp + 1), np.int32)
        ctx.check(ctx.L.pslam_peac_run_batch(ctx.h, depth.ctypes.data, B, labels.ctypes.data, planes.ctypes.data, npl.ctypes.data,
                                             midx.ctypes.data, moff.ctypes.data))
        out = []
        for f in range(B):
            n = int(npl[f])
            out.append((labels[f], planes[f, :n].copy(), [midx[f, moff[f, k]:moff[f, k + 1]].copy() for k in range(n)]))
        return out

    def vertex(self, pix: int) -> np.ndarray:
        """cloud.vertices[pix] of the reference (double), recomputed on demand."""
        h, w = self._depth.shape
        i, j = divmod(int(pix), w)
        z = float(self._depth[i, j]) * float(self._scale)
        K = self._K
        return np.array([(j - float(K[0, 2])) * z / float(K[0, 0]), (i - float(K[1, 2])) * z / float(K[1, 1]), z])

    # stage outputs for parity tests
    def debug_blocks(self, frame: int = 0):
        ctx = self._ctx
        nb = ctx.L.pslam_peac_num_blocks(ctx.h)
        st, geo = np.zeros((nb, 9)), np.zeros((nb, 8))
        n, valid = np.zeros(nb, np.int32), np.zeros(nb, np.uint8)
        ctx.check(ctx.L.pslam_peac_debug_blocks(ctx.h, frame, st.ctypes.data, geo.ctypes.data, n.ctypes.data, valid.ctypes.data))
        return st, geo, n, valid

    def debug_coarse(self, frame: int = 0):
        import ctypes as C
        ctx = self._ctx
        nb = ctx.L.pslam_peac_num_blocks(ctx.h)
        bm = np.zeros(nb, np.int32)
        nc = C.c_int32()
        ctx.check(ctx.L.pslam_peac_debug_coarse(ctx.h, frame, bm.ctypes.data, C.byref(nc)))
        return bm, nc.value


def ComputePlanes(ctx: Context, depth: np.ndarray, dist_th: float = 0.05, normals: bool = True):
    """void Frame::ComputePlanes(...) (src/Frame.cc:647-753) for a batch of depth images [B,H,W] uint16: PEAC + voxel grid + distance check + RANSAC refit +
    integral-image surface normals (include/pslam_abi.h pslam_compute_planes_batch).  The context must carry the camera (fx, fy, cx, cy, depth_scale).
    Returns per frame dict(src int32 [n], coef float32 [n][4] = mvPlaneCoefficients, points = list of float32 [k][3] = mvPlanePoints, normals float32 [m][8])."""
    import ctypes as C
    d = np.ascontiguousarray(depth, np.uint16)
    B = len(d)
    L = ctx.L
    L.pslam_compute_planes_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_float] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
    maxp, cap, nsn = int(L.pslam_peac_max_planes(ctx.h)), 16384, int(L.pslam_surface_normals_count(ctx.h))
    nk, src, coef = np.zeros(B, np.int32), np.zeros((B, maxp), np.int32), np.zeros((B, maxp, 4), np.float32)
    off, pts = np.zeros((B, maxp + 1), np.int32), np.zeros((B, cap, 3), np.float32)
    sn = np.zeros((B, nsn, 8), np.float32) if normals else None
    ctx.check(L.pslam_compute_planes_batch(ctx.h, d.ctypes.data, B, dist_th, nk.ctypes.data, src.ctypes.data, coef.ctypes.data, off.ctypes.data, pts.ctypes.data, cap,
                                           sn.ctypes.data if normals else None))
    out = []
    for f in range(B):
        n = int(nk[f])
        out.append(dict(src=src[f, :n].copy(), coef=coef[f, :n].copy(), points=[pts[f, off[f, k]:off[f, k + 1]].copy() for k in range(n)],
                        normals=sn[f].copy() if normals else None))
    return out


def UpdateMapPlanePoints(ctx: Context, jobs, cap: int | None = None):
    """void MapPlane::UpdateCoefficientsAndPoints() / (const Frame&, int id) (src/MapPlane.cc:298-365) for a batch of map planes.  jobs: one list per map plane of
    (points float32 [k][3], T float64 [4][4]) pairs - the observations' KeyFrame::mvPlanePoints[id] with the key frame's inverse pose (for the second overload
    the frame's cloud with its inverse pose and the plane's current cloud with the identity).  Returns the new mvPlanePoints per map plane (float32 [n][3],
    voxel centroids of the 0.1 m grid in ascending voxel index)."""
    import ctypes as C
    L = ctx.L
    L.pslam_map_plane_update_batch.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_void_p, C.c_void_p]
    cap = int(cap or L.pslam_map_plane_max_points(ctx.h))
    job_off, cloud_off, pts, Ts = [0], [0], [], []
    for clouds in jobs:
        for p, T in clouds:
            p = np.ascontiguousarray(p, np.float32).reshape(-1, 3)
            pts.append(p); Ts.append(np.ascontiguousarray(T, np.float64).reshape(16)); cloud_off.append(cloud_off[-1] + len(p))
        job_off.append(len(Ts))
    job_off, cloud_off = np.asarray(job_off, np.int32), np.asarray(cloud_off, np.int32)
    P = np.ascontiguousarray(np.concatenate(pts) if pts else np.zeros((0, 3), np.float32))
    T = np.ascontiguousarray(np.stack(Ts) if Ts else np.zeros((0, 16)))
    out, n = np.zeros((max(len(jobs), 1), cap, 3), np.float32), np.zeros(max(len(jobs), 1), np.int32)
    ctx.check(L.pslam_map_plane_update_batch(ctx.h, len(jobs), job_off.ctypes.data, cloud_off.ctypes.data, P.ctypes.data, T.ctypes.data, cap, out.ctypes.data,
                                             n.ctypes.data))
    return [out[j, :n[j]].copy() for j in range(len(jobs))]
