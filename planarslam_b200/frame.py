"""Python mirrors of the per-frame Frame:: helpers that sit between feature extraction and matching, on top of the C ABI."""
from __future__ import annotations

import numpy as np

from ._lib import Context


def ComputeStereoFromRGBD(ctx: Context, keys: np.ndarray, n, depth: np.ndarray, depth_factor: float, bf: float, keys_un: np.ndarray | None = None):
    """void Frame::ComputeStereoFromRGBD(const cv::Mat& imDepth) (src/Frame.cc:603-621) for a batch.
    keys: pslam_keypoint records [nframes][cap] (as ORBextractor returns them, padded), n [nframes]; depth uint16 [nframes][h][w] raw.
    Returns (mvuRight, mvDepth), float32 [nframes][cap]."""
    k = np.ascontiguousarray(keys)
    assert k.ndim == 2 and k.dtype.itemsize == 28
    nframes, cap = k.shape
    ku = k if keys_un is None else np.ascontiguousarray(keys_un)
    nn = np.ascontiguousarray(np.broadcast_to(np.asarray(n, np.int32), (nframes,)))
    d = np.ascontiguousarray(depth, np.uint16).reshape(nframes, ctx.cfg.height, ctx.cfg.width)
    ur, dz = np.zeros((nframes, cap), np.float32), np.zeros((nframes, cap), np.float32)
    ctx.check(ctx.L.pslam_compute_stereo_from_rgbd_batch(ctx.h, k.ctypes.data, ku.ctypes.data, nn.ctypes.data, cap, d.ctypes.data, nframes, float(depth_factor), float(bf),
                                                         ur.ctypes.data, dz.ctypes.data))
    return ur, dz


class FrameOutputs(object):
    """Host buffers of pslam_frame_construct_batch for `nframes` frames (page-locked when `pinned`, through torch - plumbing only), or, with `device`, CUDA
    tensors for pslam_frame_construct_batch_dev: the same fields, numeric arrays with their own dtype and records (keys, keylines, lines3d) as uint8 tensors
    with the record bytes as last dimension (view them on the host with .cpu().numpy().view(DTYPE)[..., 0])."""

    def __init__(self, ctx: Context, nframes: int, max_lines: int = 40, cap_plane_pts: int = 4096, normals: bool = True, pinned: bool = False, device=None):
        import ctypes as C
        from ._lib import KEYPOINT_DTYPE
        from .lines import KEYLINE_DTYPE, LINE3D_DTYPE
        L = ctx.L
        capk, maxp, nsn = int(L.pslam_orb_max_keypoints(ctx.h)), int(L.pslam_peac_max_planes(ctx.h)), int(L.pslam_surface_normals_count(ctx.h))
        self._keep = []
        assert not (pinned and device is not None), "pinned host buffers or device buffers, not both"

        def buf(shape, dtype):
            if device is not None:
                import torch
                dt = np.dtype(dtype)
                if dt.names is not None:
                    return torch.zeros(tuple(shape) + (dt.itemsize,), dtype=torch.uint8, device=device)
                return torch.zeros(tuple(shape), dtype=getattr(torch, dt.name), device=device)
            if not pinned:
                return np.zeros(shape, dtype)
            import torch
            t = torch.zeros(int(np.prod(shape)) * np.dtype(dtype).itemsize, dtype=torch.uint8).pin_memory()
            self._keep.append(t)
            return t.numpy().view(dtype).reshape(shape)
        self.keys, self.desc, self.n_keys = buf((nframes, capk), KEYPOINT_DTYPE), buf((nframes, capk, 32), np.uint8), buf((nframes,), np.int32)
        self.u_right, self.depth_kp = buf((nframes, capk), np.float32), buf((nframes, capk), np.float32)
        self.keylines, self.line_functions = buf((nframes, max_lines), KEYLINE_DTYPE), buf((nframes, max_lines, 3), np.float64)
        self.line_desc, self.lines3d = buf((nframes, max_lines, 32), np.uint8), buf((nframes, max_lines), LINE3D_DTYPE)
        self.n_lines, self.n_rand_drawn = buf((nframes,), np.int32), buf((nframes,), np.int32)
        self.n_planes, self.plane_src, self.plane_coef = buf((nframes,), np.int32), buf((nframes, maxp), np.int32), buf((nframes, maxp, 4), np.float32)
        self.plane_pt_off, self.plane_pts = buf((nframes, maxp + 1), np.int32), buf((nframes, cap_plane_pts, 3), np.float32)
        self.surface_normals8 = buf((nframes, nsn, 8), np.float32) if normals else None
        self.nframes, self.max_lines, self.cap_plane_pts = nframes, max_lines, cap_plane_pts

        class _S(C.Structure):
            _fields_ = [(n, C.c_void_p) for n in ("keys", "desc", "n_keys", "u_right", "depth_kp", "keylines", "line_functions", "line_desc", "lines3d", "n_lines",
                                                  "n_rand_drawn", "n_planes", "plane_src", "plane_coef", "plane_pt_off", "plane_pts")] + \
                       [("cap_plane_pts", C.c_int32), ("surface_normals8", C.c_void_p)]
        s = _S()
        for n, _ in _S._fields_:
            if n == "cap_plane_pts":
                s.cap_plane_pts = cap_plane_pts
            else:
                a = getattr(self, n)
                setattr(s, n, None if a is None else a.data_ptr() if device is not None else a.ctypes.data)
        self.struct = s

    def nbytes(self) -> int:
        return sum(a.nbytes for a in (self.keys, self.desc, self.n_keys, self.u_right, self.depth_kp, self.keylines, self.line_functions, self.line_desc, self.lines3d,
                                      self.n_lines, self.n_rand_drawn, self.n_planes, self.plane_src, self.plane_coef, self.plane_pt_off, self.plane_pts) if a is not None) + \
            (self.surface_normals8.nbytes if self.surface_normals8 is not None else 0)


def ConstructFrames(ctx: Context, gray, depth, out: FrameOutputs | None = None, depth_factor: float | None = None, bf: float = 40.0, plane_dist_th: float = 0.05,
                    line_seed: int = 1, nframes: int | None = None) -> FrameOutputs:
    """The compute of Frame::Frame(imRGB, imGray, imDepth, ...) (src/Frame.cc:55-140) for a batch: ExtractORB + ComputeStereoFromRGBD, ExtractLSD (LBD, isLineGood),
    ComputePlanes, with ONE upload of the frames (include/pslam_abi.h pslam_frame_construct_batch).  gray uint8 [B][h][w], depth uint16 [B][h][w] (numpy arrays, or
    integers = addresses of host buffers together with nframes)."""
    import ctypes as C
    L = ctx.L
    L.pslam_frame_construct_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int, C.c_uint32, C.c_void_p]
    if isinstance(gray, np.ndarray):
        g, d = np.ascontiguousarray(gray, np.uint8), np.ascontiguousarray(depth, np.uint16)
        nframes = len(g)
        gp, dp = g.ctypes.data, d.ctypes.data
    else:
        gp, dp = int(gray), int(depth)
    out = out or FrameOutputs(ctx, nframes)
    df = float(ctx.cfg.depth_scale) if depth_factor is None else float(depth_factor)
    ctx.check(L.pslam_frame_construct_batch(ctx.h, gp, dp, nframes, df, float(bf), float(plane_dist_th), out.max_lines, line_seed, C.byref(out.struct)))
    return out


def _cuda_input(ctx: Context, t, name: str, dtypes, ndims):
    """t as a contiguous CUDA tensor on the context's device, [B][height][width] (+ a channel dimension of 3 or 4 when 4 in ndims)."""
    import torch
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
        raise TypeError(f"{name}: a CUDA tensor is required, got {type(t).__name__}" + (f" on {t.device}" if isinstance(t, torch.Tensor) else ""))
    if t.device.index != ctx.cfg.device:
        raise ValueError(f"{name}: tensor on {t.device}, the context runs on cuda:{ctx.cfg.device}")
    if t.dtype not in dtypes:
        raise TypeError(f"{name}: dtype {t.dtype} is not one of {', '.join(str(d) for d in dtypes)}")
    if t.dim() not in ndims or tuple(t.shape[1:3]) != (ctx.cfg.height, ctx.cfg.width) or (t.dim() == 4 and t.shape[3] not in (3, 4)):
        raise ValueError(f"{name}: shape {tuple(t.shape)} is not [B, {ctx.cfg.height}, {ctx.cfg.width}]" + (" (+ [3|4])" if 4 in ndims else ""))
    return t.contiguous()


CUDA_STREAM_LEGACY = 1     # cudaStreamLegacy: torch's default stream has the handle 0, which pslam_set_stream reads as "the context's own stream"


def _on_current_stream(ctx: Context, t) -> None:
    """Point the context at torch.cuda.current_stream() on t's device (the context's own stream does not wait for torch's default stream)."""
    import torch
    ctx.set_stream(torch.cuda.current_stream(t.device).cuda_stream or CUDA_STREAM_LEGACY)


def gray_from_color(ctx: Context, image, rgb: bool = True):
    """The cvtColor of Tracking::GrabImageRGBD (src/Tracking.cc:157-172) on device frames: CUDA uint8 [B][h][w][3|4] -> uint8 [B][h][w], bit-exact to
    OpenCV 4.13's RGB2GRAY / BGR2GRAY / RGBA2GRAY / BGRA2GRAY; rgb = Camera.RGB (True: R first).  Enqueued on torch.cuda.current_stream(), which the context
    keeps using afterwards (pslam_gray_from_color_batch_dev)."""
    import torch
    img = _cuda_input(ctx, image, "image", (torch.uint8,), (4,))
    out = torch.empty(img.shape[:3], dtype=torch.uint8, device=img.device)
    _on_current_stream(ctx, img)
    ctx.check(ctx.L.pslam_gray_from_color_batch_dev(ctx.h, img.data_ptr(), int(img.shape[3]), 1 if rgb else 0, int(img.shape[0]), out.data_ptr()))
    return out


def construct_frames_dev(ctx: Context, image, depth, *, rgb: bool = True, depth_factor: float | None = None, bf: float = 40.0, plane_dist_th: float = 0.05,
                         line_seed: int = 1, max_lines: int = 40, cap_plane_pts: int = 4096, normals: bool = True, out: FrameOutputs | None = None) -> FrameOutputs:
    """The compute of Frame::Frame(imRGB, imGray, imDepth, ...) (src/Frame.cc:55-140) on frames already on the GPU (pslam_frame_construct_batch_dev): the
    same products as ConstructFrames, as CUDA tensors (FrameOutputs with device=...), plus `status` int32 [B]: the PSLAM_FRAME_CAP_* bits per frame (0: no
    capacity was exceeded).  image: CUDA uint8 [B][h][w] grey, or [B][h][w][3|4] colour, converted first as GrabImageRGBD does (rgb = Camera.RGB); depth:
    CUDA uint16 (or int16 holding the same bits) [B][h][w].  Enqueued on torch.cuda.current_stream() without a host synchronisation; `out` (device
    FrameOutputs for B frames) replaces max_lines / cap_plane_pts / normals."""
    import ctypes as C
    import torch
    img = _cuda_input(ctx, image, "image", (torch.uint8,), (3, 4))
    d = _cuda_input(ctx, depth, "depth", (torch.uint16, torch.int16), (3,))
    if d.device != img.device or d.shape[0] != img.shape[0]:
        raise ValueError(f"depth {tuple(d.shape)} on {d.device} does not match image {tuple(img.shape)} on {img.device}")
    B = int(img.shape[0])
    gray = gray_from_color(ctx, img, rgb) if img.dim() == 4 else img
    out = out or FrameOutputs(ctx, B, max_lines, cap_plane_pts, normals, device=img.device)
    out.status = torch.empty(B, dtype=torch.int32, device=img.device)
    df = float(ctx.cfg.depth_scale) if depth_factor is None else float(depth_factor)
    _on_current_stream(ctx, img)
    ctx.check(ctx.L.pslam_frame_construct_batch_dev(ctx.h, gray.data_ptr(), d.data_ptr(), B, df, float(bf), float(plane_dist_th), out.max_lines, line_seed,
                                                    C.byref(out.struct), out.status.data_ptr()))
    return out
