"""GPU: the Frame constructor on device-resident frames (pslam_frame_construct_batch_dev, construct_frames_dev) writes the bytes the host-pointer call
pslam_frame_construct_batch writes, at every camera and image size of depth_cameras.CASES, and reports per frame, in its status word, exactly the capacity
overflows the host call turns into PSLAM_E_CAPACITY; the colour conversion of Tracking::GrabImageRGBD (src/Tracking.cc:157-172, k_gray_from_color) equals
the CPU oracle cvtcolor_oracle.py, which is pinned to cv2 4.13 on every (R, G, B) triple (test_oracle_gray_from_color.py).  The host call is itself
held to the separate calls and the oracle by test_frame_construct_gpu.py and test_depth_products_cameras_gpu.py."""
import ctypes as C

import numpy as np
import pytest

import cvtcolor_oracle
from depth_cameras import CASES, frames, scale_of

pytestmark = pytest.mark.gpu
B, FLAT, ZERO = 5, 1, 2
BF, CAP_PTS = 40.0, 16384


def _ctx(case, n=B):
    from planarslam_b200._lib import Context
    w, h, K, factor, kw = CASES[case]
    return Context(w, h, max_batch=n, fx=K[0], fy=K[1], cx=K[2], cy=K[3], depth_scale=scale_of(factor), **kw)


def _inputs(case):
    gray, depth = frames(case, B, zero_slot=ZERO)
    gray[FLAT] = 128
    return gray, depth


def _host(ctx, gray, depth, cap_pts=CAP_PTS):
    """pslam_frame_construct_batch: (return code, FrameOutputs)."""
    from planarslam_b200.frame import FrameOutputs
    out = FrameOutputs(ctx, len(gray), cap_plane_pts=cap_pts)
    ctx.L.pslam_frame_construct_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int, C.c_uint32, C.c_void_p]
    rc = ctx.L.pslam_frame_construct_batch(ctx.h, gray.ctypes.data, depth.ctypes.data, len(gray), float(ctx.cfg.depth_scale), BF, 0.05, out.max_lines, 1,
                                           C.byref(out.struct))
    return rc, out


def _dev_tensors(gray, depth):
    import torch
    return torch.from_numpy(gray).cuda(), torch.from_numpy(depth.view(np.int16)).cuda()


def _to_host(t, dtype):
    a = t.cpu().numpy()
    return a.view(dtype)[..., 0] if np.dtype(dtype).names else a


def assert_same_products(host, dev, normals=True, drawn=True):
    """Every valid entry of the device outputs equals the host outputs byte for byte (padding beyond the counts is not part of the products)."""
    from planarslam_b200._lib import KEYPOINT_DTYPE
    from planarslam_b200.lines import KEYLINE_DTYPE, LINE3D_DTYPE
    d = {n: _to_host(getattr(dev, n), dt) for n, dt in [("keys", KEYPOINT_DTYPE), ("keylines", KEYLINE_DTYPE), ("lines3d", LINE3D_DTYPE)]}
    for n in ("desc", "n_keys", "u_right", "depth_kp", "line_functions", "line_desc", "n_lines", "n_rand_drawn", "n_planes", "plane_src", "plane_coef",
              "plane_pt_off", "plane_pts") + (("surface_normals8",) if normals else ()):
        d[n] = getattr(dev, n).cpu().numpy()
    for n in ("n_keys", "n_lines", "n_planes") + (("n_rand_drawn",) if drawn else ()):
        assert np.array_equal(d[n], getattr(host, n)), n
    for f in range(host.nframes):
        k, m, p = int(host.n_keys[f]), int(host.n_lines[f]), int(host.n_planes[f])
        for n in ("keys", "desc", "u_right", "depth_kp"):
            assert d[n][f, :k].tobytes() == getattr(host, n)[f, :k].tobytes(), (f, n)
        for n in ("keylines", "line_functions", "line_desc", "lines3d"):
            assert d[n][f, :m].tobytes() == getattr(host, n)[f, :m].tobytes(), (f, n)
        for n in ("plane_src", "plane_coef"):
            assert d[n][f, :p].tobytes() == getattr(host, n)[f, :p].tobytes(), (f, n)
        assert np.array_equal(d["plane_pt_off"][f, :p + 1], host.plane_pt_off[f, :p + 1]), f
        npts = min(int(host.plane_pt_off[f, p]), host.cap_plane_pts)
        assert d["plane_pts"][f, :npts].tobytes() == host.plane_pts[f, :npts].tobytes(), f
    if normals:
        assert d["surface_normals8"].tobytes() == host.surface_normals8.tobytes()


@pytest.mark.parametrize("case", sorted(CASES))
def test_dev_constructor_equals_the_host_call(case):
    import torch
    from planarslam_b200.frame import FrameOutputs, construct_frames_dev
    gray, depth = _inputs(case)
    ctx = _ctx(case)
    rc, host = _host(ctx, gray, depth)
    assert rc == 0, ctx.L.pslam_last_error(ctx.h)
    assert host.n_keys[FLAT] == 0 and host.n_planes[ZERO] == 0 and host.n_keys.max() > 0
    w, h = CASES[case][:2]
    if w * h >= 320 * 240:          # PEAC finds no plane in the 120x117 frames
        assert host.n_planes.max() > 0
    g, d = _dev_tensors(gray, depth)
    dctx = _ctx(case)
    on = construct_frames_dev(dctx, g, d, bf=BF, plane_dist_th=0.05, line_seed=1, cap_plane_pts=CAP_PTS, normals=True)
    # normals off and n_rand_drawn NULL
    o2 = FrameOutputs(dctx, B, cap_plane_pts=CAP_PTS, normals=False, device=g.device)
    o2.struct.n_rand_drawn = None
    off = construct_frames_dev(dctx, g, d, bf=BF, plane_dist_th=0.05, line_seed=1, out=o2)
    torch.cuda.synchronize()
    assert on.status.cpu().numpy().tolist() == [0] * B and off.status.cpu().numpy().tolist() == [0] * B
    assert_same_products(host, on)
    assert_same_products(host, off, normals=False, drawn=False)
    assert not off.n_rand_drawn.any().item()        # not written when NULL


def test_plane_point_overflow_sets_the_status_bit_where_the_host_call_fails():
    import torch
    from planarslam_b200._lib import E_CAPACITY, FRAME_CAP_PLANE_PTS as bit
    from planarslam_b200.frame import construct_frames_dev
    case = "tum3"
    gray, depth = _inputs(case)
    ctx = _ctx(case)
    _, full = _host(ctx, gray, depth)
    totals = np.array([full.plane_pt_off[f, full.n_planes[f]] for f in range(B)])
    cap = int(totals[totals > 0].min())                   # the smallest non-empty frame just fits, larger ones overflow
    over = [_host(ctx, gray[f:f + 1], depth[f:f + 1], cap)[0] == E_CAPACITY for f in range(B)]
    assert any(over) and not all(over), totals
    rc, host = _host(ctx, gray, depth, cap)
    assert rc == E_CAPACITY
    g, d = _dev_tensors(gray, depth)
    dev = construct_frames_dev(_ctx(case), g, d, bf=BF, plane_dist_th=0.05, line_seed=1, cap_plane_pts=cap)
    torch.cuda.synchronize()
    st = dev.status.cpu().numpy()
    assert [bool(s & bit) for s in st] == over and not (st & ~bit).any(), (st, over)
    assert_same_products(host, dev)


def _color(gray: np.ndarray, alpha: bool, seed: int) -> np.ndarray:
    """A colour frame batch derived from grey renders: three different channels (and a noise alpha), so that the channel order matters."""
    rng = np.random.default_rng(seed)
    noise = rng.integers(0, 256, gray.shape, dtype=np.uint8)
    ch = [gray, (gray.astype(np.uint16) * 3 // 4 + noise // 4).astype(np.uint8), 255 - gray]
    if alpha:
        ch.append(rng.integers(0, 256, gray.shape, dtype=np.uint8))
    return np.ascontiguousarray(np.stack(ch, -1))


def test_gray_from_color_equals_the_oracle_on_every_triple():
    import torch
    from planarslam_b200._lib import Context
    from planarslam_b200.frame import gray_from_color
    v = np.arange(1 << 24, dtype=np.uint32)
    rgb3 = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8).reshape(256, 256, 256, 3)
    alpha = np.random.default_rng(5).integers(0, 256, rgb3.shape[:3] + (1,), dtype=np.uint8)
    ctx = Context(256, 256, 256, nlevels=4)
    for img in (rgb3, np.concatenate([rgb3, alpha], -1)):
        t = torch.from_numpy(img).cuda()
        for rgb in (True, False):
            got = gray_from_color(ctx, t, rgb).cpu().numpy()
            assert np.array_equal(got, cvtcolor_oracle.gray_from_color(img, rgb)), (img.shape[-1], rgb)


@pytest.mark.parametrize("case", ["odd_644x482", "min_120x117"])
def test_gray_from_color_on_renders(case):
    import torch
    from planarslam_b200.frame import gray_from_color
    gray, _ = frames(case, 3)
    ctx = _ctx(case, 3)
    for ch in (3, 4):
        img = _color(gray, ch == 4, seed=ch)
        for rgb in (True, False):
            got = gray_from_color(ctx, torch.from_numpy(img).cuda(), rgb).cpu().numpy()
            assert np.array_equal(got, cvtcolor_oracle.gray_from_color(img, rgb)), (ch, rgb)


def test_color_frames_equal_the_host_call_on_the_oracle_grey():
    import torch
    from planarslam_b200.frame import construct_frames_dev
    case = "tum3"
    gray, depth = _inputs(case)
    ctx = _ctx(case)
    for ch, rgb in ((3, True), (4, False)):
        img = _color(gray, ch == 4, seed=10 + ch)
        rc, host = _host(ctx, cvtcolor_oracle.gray_from_color(img, rgb), depth)
        assert rc == 0
        _, d = _dev_tensors(gray, depth)
        dev = construct_frames_dev(ctx, torch.from_numpy(img).cuda(), d, rgb=rgb, bf=BF, plane_dist_th=0.05, line_seed=1, cap_plane_pts=CAP_PTS)
        torch.cuda.synchronize()
        assert not dev.status.any().item()
        assert host.n_keys.max() > 0 and host.n_lines.max() > 0
        assert_same_products(host, dev)


def test_dev_call_only_enqueues():
    """After a warm-up call (which sizes the scratch), a call behind a long sleep on a side stream returns before the stream has run it; its results are
    those of the warm-up once the stream is synchronised."""
    import torch
    from planarslam_b200.frame import construct_frames_dev
    case = "tum3"
    gray, depth = _inputs(case)
    g, d = _dev_tensors(gray, depth)
    ctx = _ctx(case)
    kw = dict(bf=BF, plane_dist_th=0.05, line_seed=1, cap_plane_pts=CAP_PTS)
    warm = construct_frames_dev(ctx, g, d, **kw)
    torch.cuda.synchronize()
    rc, host = _host(_ctx(case), gray, depth)
    assert rc == 0
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(2_000_000_000)          # about a second at H100 clocks
        out = construct_frames_dev(ctx, g, d, **kw)
        pending = not s.query()
    assert pending, "the call waited for the stream"
    s.synchronize()
    assert not out.status.any().item() and not warm.status.any().item()
    assert_same_products(host, out)
    # torch's default stream (handle 0): the call queues behind the sleep as well, so reading the outputs, which waits for that stream only, sees them
    torch.cuda._sleep(1_000_000_000)
    assert_same_products(host, construct_frames_dev(ctx, g, d, **kw))


def test_invalid_arguments():
    import torch
    from planarslam_b200._lib import E_INVALID
    from planarslam_b200.frame import FrameOutputs, construct_frames_dev, gray_from_color
    case = "min_120x117"
    w, h = CASES[case][0], CASES[case][1]
    ctx = _ctx(case)
    L = ctx.L
    buf = torch.zeros(B * h * w * 4 + 16, dtype=torch.uint8, device="cuda")
    gray = torch.zeros(B * h * w + 16, dtype=torch.uint8, device="cuda")
    depth = torch.zeros(B * h * w + 16, dtype=torch.int16, device="cuda")
    col, gp, dp = buf.data_ptr(), gray.data_ptr(), depth.data_ptr()
    assert L.pslam_gray_from_color_batch_dev(ctx.h, col, 3, 1, B, gp) == 0
    for args in ((col + 1, 3, 1, B, gp), (col, 3, 1, B, gp + 2), (col, 5, 1, B, gp), (col, 1, 1, B, gp), (col, 3, 1, 0, gp), (col, 3, 1, B + 1, gp),
                 (None, 3, 1, B, gp), (col, 4, 1, B, None)):
        assert L.pslam_gray_from_color_batch_dev(ctx.h, *args) == E_INVALID, args
    out = FrameOutputs(ctx, B, cap_plane_pts=1024, device="cuda")
    status = torch.zeros(B, dtype=torch.int32, device="cuda")
    sp = status.data_ptr()

    def call(g, d, n, o=out, st=sp):
        return L.pslam_frame_construct_batch_dev(ctx.h, g, d, n, float(ctx.cfg.depth_scale), BF, 0.05, 40, 1, C.byref(o.struct) if o else None, st)
    for args in ((gp + 1, dp, B), (gp + 2, dp, B), (gp, dp + 2, B), (gp, dp, 0), (gp, dp, B + 1), (None, dp, B), (gp, None, B)):
        assert call(*args) == E_INVALID, args
    assert call(gp, dp, B, o=None) == E_INVALID and call(gp, dp, B, st=None) == E_INVALID
    out.struct.keys = None
    assert call(gp, dp, B) == E_INVALID
    torch.cuda.synchronize()
    # the Python layer rejects what the ABI cannot see
    g3, d3 = gray[:B * h * w].view(B, h, w), depth[:B * h * w].view(B, h, w)
    with pytest.raises(TypeError):
        construct_frames_dev(ctx, g3.cpu(), d3)
    with pytest.raises(TypeError):
        construct_frames_dev(ctx, g3, d3.float())
    with pytest.raises(ValueError):
        construct_frames_dev(ctx, g3[:, :, :w - 4].contiguous(), d3)
    with pytest.raises(ValueError):
        gray_from_color(ctx, buf[:B * h * w * 2].view(B, h, w, 2))
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError):
            construct_frames_dev(ctx, g3.to("cuda:1"), d3.to("cuda:1"))
