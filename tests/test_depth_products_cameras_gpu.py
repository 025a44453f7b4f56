"""GPU: the depth half of the RGB-D Frame constructor - ComputePlanes' post-processing and surface normals (k_planes_post, k_sn_*), ComputeStereoFromRGBD
and isLineGood - at every camera and image size of depth_cameras.CASES (TUM3, ICL with fy < 0, TUM2 with DepthMapFactor 5208, TAMU, the 1280x960 bench
configuration, odd sub-sampled grids, the smallest frames), against the CPU oracle; and the edges of the exact voxel sums: carries on every axis of a
voxel with ~270 k members, and the key range of the voxel table (+-51.2 m sideways, 409.6 m deep).

Bar (as test_planepost_gpu.py / test_line3d_gpu.py / test_frame_construct_gpu.py): the same planes kept, voxel clouds bit-exact, coefficients to 2e-5,
normals bit-exact with the NaN pattern, stereo and 3-D lines bit-exact with the same rand() draw counts, the one-call Frame constructor equal to the
separate calls.  Each batch has an odd number of frames (the four-frames-per-CTA normal kernels end on a partial CTA), an all-zero depth frame in a middle
slot and a real frame in the last slot of max_batch."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib
from depth_cameras import CASES, frames, scale_of
from test_oracle_surface_normals_independent import voxel_centroids

pytestmark = pytest.mark.gpu
f32 = np.float32
B, ZERO = 5, 2
BF = 40.0


def _ctx(w, h, n, K, scale, **kw):
    from planarslam_b200._lib import Context
    return Context(w, h, max_batch=n, fx=K[0], fy=K[1], cx=K[2], cy=K[3], depth_scale=scale, **kw)


def _check_planes(res, depth, K, scale):
    kept = 0
    for f in range(len(depth)):
        o = oracle_lib.planes_post(depth[f], K, f32(scale))
        r = res[f]
        assert [p["src"] for p in o] == r["src"].tolist(), f
        for k, p in enumerate(o):
            assert np.array_equal(r["points"][k], p["points"]), (f, k)
            assert np.abs(r["coef"][k] - p["coef"]).max() < 2e-5, (f, k, r["coef"][k], p["coef"])
        kept += len(o)
    return kept


@pytest.mark.parametrize("case", sorted(CASES))
def test_depth_products_match_the_oracle(case):
    from planarslam_b200._lib import KEYPOINT_DTYPE
    from planarslam_b200.frame import ComputeStereoFromRGBD, ConstructFrames, FrameOutputs
    from planarslam_b200.lines import LineSegment, isLineGood
    from planarslam_b200.planes import ComputePlanes
    w, h, K, factor, kw = CASES[case]
    scale = scale_of(factor)
    gray, depth = frames(case, B, zero_slot=ZERO)
    ctx = _ctx(w, h, B, K, scale, **kw)
    L = ctx.L
    # ComputePlanes: plane post-processing and surface normals
    res = ComputePlanes(ctx, depth, 0.05, normals=True)
    kept = _check_planes(res, depth, K, scale)
    assert len(res[ZERO]["src"]) == 0
    if w * h >= 320 * 240:
        assert kept >= B + 1
    n_sn = int(L.pslam_surface_normals_count(ctx.h))
    assert n_sn == (((w + 2) // 3) // 2) * (((h + 2) // 3) // 2)
    for f in range(B):
        osn = oracle_lib.surface_normals(depth[f], K, f32(scale))
        sn = res[f]["normals"]
        assert sn.shape == osn.shape == (n_sn, 8), f
        assert np.array_equal(sn, osn, equal_nan=True), f
        assert np.isnan(sn[:, :3]).all() == (f == ZERO), f
    # ComputeStereoFromRGBD on the key points the GPU ORB returns
    cap = int(L.pslam_orb_max_keypoints(ctx.h))
    kps, desc, nk = np.zeros((B, cap), KEYPOINT_DTYPE), np.zeros((B, cap, 32), np.uint8), np.zeros(B, np.int32)
    ctx.check(L.pslam_orb_extract_batch(ctx.h, gray.ctypes.data, B, kps.ctypes.data, desc.ctypes.data, cap, nk.ctypes.data))
    assert nk.min() > 50
    ur, dz = ComputeStereoFromRGBD(ctx, kps, nk, depth, scale, BF)
    depth_m = depth.astype(f32) * f32(scale)
    for f in range(B):
        k = kps[f, :nk[f]]
        xy = np.ascontiguousarray(np.stack([k["x"], k["y"]], 1), f32)
        our, odz = oracle_lib.compute_stereo_from_rgbd(xy, xy, depth_m[f], BF)
        assert np.array_equal(ur[f, :nk[f]], our) and np.array_equal(dz[f, :nk[f]], odz), f
        assert (dz[f, :nk[f]] > 0).any() == (f != ZERO)
    # isLineGood on the key lines the GPU LSD returns
    lines = LineSegment(ctx=ctx).ExtractLineSegmentWithDescriptors(gray, 40)
    from planarslam_b200.lines import KEYLINE_DTYPE
    kl, nl = np.zeros((B, 40), KEYLINE_DTYPE), np.array([len(x[0]) for x in lines], np.int32)
    for f in range(B):
        kl[f, :nl[f]] = lines[f][0]
    assert nl.min() >= (5 if w >= 320 else 1)
    out3, drawn = isLineGood(ctx, kl, nl, depth, K, scale, seed=1)
    for f in range(B):
        o = oracle_lib.lines3d_frame(kl[f, :nl[f]], depth_m[f], K, seed=1)
        g = out3[f, :nl[f]]
        assert drawn[f] == o["n_drawn"], f
        assert np.array_equal(g["valid"], o["valid"]) and np.array_equal(g["n_points"], o["n_points"]), f
        assert np.array_equal(g["inliers"], o["inliers"]) and np.array_equal(g["n_inliers"], o["n_inliers"]), f
        assert np.array_equal(np.concatenate([g["A"], g["B"]], 1), o["lines3d"]) and np.array_equal(g["depth"], o["depth_line"]), f
        assert np.array_equal(g["director"], o["director"], equal_nan=True), f
        assert not g["valid"].any() or f != ZERO
    if case not in ("config5", "icl"):
        return
    # the one-call Frame constructor on a second context equals the separate calls above
    fctx = _ctx(w, h, B, K, scale, **kw)
    out = ConstructFrames(fctx, gray, depth, FrameOutputs(fctx, B, cap_plane_pts=16384), depth_factor=scale, bf=BF, plane_dist_th=0.05, line_seed=1)
    assert np.array_equal(out.n_keys, nk)
    for f in range(B):
        n = nk[f]
        assert np.array_equal(out.keys[f, :n], kps[f, :n]) and np.array_equal(out.desc[f, :n], desc[f, :n]), f
        assert np.array_equal(out.u_right[f, :n], ur[f, :n]) and np.array_equal(out.depth_kp[f, :n], dz[f, :n]), f
        m = nl[f]
        assert out.n_lines[f] == m
        assert out.keylines[f, :m].tobytes() == kl[f, :m].tobytes() and np.array_equal(out.line_functions[f, :m], lines[f][1]), f
        assert np.array_equal(out.line_desc[f, :m], lines[f][2]), f
        assert out.lines3d[f, :m].tobytes() == out3[f, :m].tobytes() and out.n_rand_drawn[f] == drawn[f], f
        p = res[f]
        k = len(p["src"])
        assert out.n_planes[f] == k
        assert np.array_equal(out.plane_src[f, :k], p["src"]) and np.array_equal(out.plane_coef[f, :k], p["coef"]), f
        for q in range(k):
            assert np.array_equal(out.plane_pts[f, out.plane_pt_off[f, q]:out.plane_pt_off[f, q + 1]], p["points"][q]), (f, q)
        assert np.array_equal(out.surface_normals8[f], p["normals"], equal_nan=True), f


def test_voxel_sums_carry_on_every_axis():
    """A frontal plane 0.199 m in front of the 1280x960 camera fills the whole image: the voxel at x, y in [-0.1, 0) holds ~267 k members, and every axis of
    its fixed-point sum, relative to the voxel base, passes 2^33 - the low 32-bit words wrap several times and the 10-bit carry fields hold the rest."""
    from planarslam_b200.planes import ComputePlanes
    w, h, K, factor, _ = CASES["config5"]
    scale = scale_of(factor)
    depth = np.full((1, h, w), 995, np.uint16)
    members = np.arange(w * h)
    v, u = np.divmod(members, w)
    zz = depth[0].ravel().astype(np.float64) * float(f32(scale))
    X = np.stack([(u - K[2]) * zz / K[0], (v - K[3]) * zz / K[1], zz], 1).astype(f32)
    idx = np.floor(X * f32(10.0)).astype(np.int64)
    rel = np.rint(X.astype(np.float64) * 2.0 ** 20).astype(np.int64) - (idx * 104857 - 1024)      # llrint(c * 2^20) - pp_base(floor(c * 10))
    assert (rel >= 0).all() and (rel < 2 ** 17).all()
    _, vox = np.unique(idx[:, 0] + 4096 * idx[:, 1] + 4096 * 4096 * idx[:, 2], return_inverse=True)
    sums = np.stack([np.bincount(vox, weights=rel[:, a].astype(np.float64)) for a in range(3)], 1)
    big = int(np.argmax(np.bincount(vox)))
    print("per-axis relative sums of the largest voxel: 2^%.2f, 2^%.2f, 2^%.2f" % tuple(np.log2(sums[big])))
    assert (sums[big] >= 2.0 ** 33).all()
    assert ((idx[vox == big] < 0) == [True, True, False]).all()                                     # negative x and y: negative voxel bases
    res = ComputePlanes(_ctx(w, h, 1, K, scale, nfeatures=2000), depth, 0.05, normals=False)
    o = oracle_lib.planes_post(depth[0], K, f32(scale))
    assert [p["src"] for p in o] == res[0]["src"].tolist() == [0]
    _, exact, count = voxel_centroids(depth[0], K, scale, members)
    assert count.max() > 260000
    assert np.array_equal(res[0]["points"][0], o[0]["points"]) and np.array_equal(res[0]["points"][0], exact)
    assert np.abs(res[0]["coef"][0] - o[0]["coef"]).max() < 2e-5


def _post_records(ctx, depth, records, cap=16384):
    """pslam_planes_post_batch_dev on caller-made plane records: records[f] = list of (normal, center, member pixel indices).  Returns (n_kept, src, coef,
    pt_off, pts, status) as numpy arrays."""
    import torch
    from planarslam_b200._lib import PLANE_DTYPE
    L = ctx.L
    L.pslam_planes_post_batch_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 4 + [C.c_float] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
    n, (H, W) = len(depth), depth.shape[1:]
    maxp = int(L.pslam_peac_max_planes(ctx.h))
    planes = np.zeros((n, maxp), PLANE_DTYPE)
    npl, midx, moff = np.zeros(n, np.int32), np.zeros((n, H * W), np.int32), np.zeros((n, maxp + 1), np.int32)
    for f, recs in enumerate(records):
        npl[f] = len(recs)
        for p, (nrm, ctr, mem) in enumerate(recs):
            planes["normal"][f, p], planes["center"][f, p], planes["N"][f, p] = nrm, ctr, len(mem)
            midx[f, moff[f, p]:moff[f, p] + len(mem)] = mem
            moff[f, p + 1:] = moff[f, p] + len(mem)
    dev = torch.device("cuda", 0)
    t = [torch.from_numpy(a).to(dev) for a in (depth.view(np.int16), planes.view(np.uint8), npl, midx, moff)]
    out = [torch.zeros(n, dtype=torch.int32, device=dev), torch.zeros((n, maxp), dtype=torch.int32, device=dev),
           torch.zeros((n, maxp, 4), dtype=torch.float32, device=dev), torch.zeros((n, maxp + 1), dtype=torch.int32, device=dev),
           torch.zeros((n, cap, 3), dtype=torch.float32, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)]
    ctx.check(L.pslam_planes_post_batch_dev(ctx.h, t[0].data_ptr(), n, *[a.data_ptr() for a in t[1:]], 0.05, *[a.data_ptr() for a in out[:5]], cap, out[5].data_ptr()))
    ctx.synchronize()
    return [a.cpu().numpy() for a in out]


WIDE_K, WIDE_SCALE = (200.0, 200.0, 319.5, 239.5), scale_of(1000.0)


def _receding_wall(x_edge, mirror):
    """A vertical wall 1 m deep at one image edge that recedes to x = x_edge (+-) at the other, seen by a 640x480 camera with fx = fy = 200 and depth
    factor 1000, as a hand-made plane record: its members are 80 rows of a near block (many pixels per voxel) and of the far column(s) within 5 m of the
    edge, so the record has ~300 voxels - far below the 2048 slots even when every member were binned."""
    W, H = 640, 480
    t = (np.arange(W) - WIDE_K[2]) / WIDE_K[0]
    zl = x_edge / t[0]
    b = (zl - 1.0) / (x_edge - t[-1])
    a = 1.0 - b * t[-1]
    depth = np.repeat(np.rint(a / (1 - b * t) * 1000).astype(np.uint16)[None], H, 0)
    normal = np.array([-b, 0.0, 1.0]) / np.hypot(b, 1.0)
    x = ((np.arange(W) - WIDE_K[2]) * (depth[0].astype(np.float64) * WIDE_SCALE) / WIDE_K[0]).astype(f32)
    cols = np.concatenate([np.arange(440, 640), np.nonzero(x < x_edge + 5.0)[0]])
    if mirror:                                                     # u -> 639 - u: x -> -x exactly (cx = 319.5)
        depth, cols, normal = depth[:, ::-1].copy(), W - 1 - cols, normal * [-1, 1, 1]
    mem = np.sort((np.arange(200, 280)[:, None] * W + cols[None]).ravel()).astype(np.int32)
    return depth, (normal, np.array([0.0, 0.0, a]), mem)


def test_voxel_key_range_sideways():
    """Members at x = -51.15 / +51.15 m (inside the +-51.2 m of the voxel keys) give exactly the oracle's plane; members at -53 / +53 m raise the capacity
    bit (32) of the frame's status, next to an unaffected frame, instead of being binned into a wrong voxel."""
    walls = [_receding_wall(-51.15, False), _receding_wall(-51.15, True), _receding_wall(-53.0, False), _receding_wall(-53.0, True)]
    depth = np.stack([d for d, _ in walls])
    ctx = _ctx(640, 480, len(walls), WIDE_K, WIDE_SCALE)
    n_kept, src, coef, off, pts, status = _post_records(ctx, depth, [[r] for _, r in walls])
    for f in (0, 1):
        nrm, ctr, mem = walls[f][1]
        v, u = np.divmod(mem, 640)
        x = ((u - WIDE_K[2]) * (depth[f].ravel()[mem] * WIDE_SCALE) / WIDE_K[0]).astype(f32)
        assert 51.1 < np.abs(x).max() < 51.2
        o = oracle_lib.planes_post_records(depth[f], np.concatenate([nrm, ctr])[None], [mem], WIDE_K, f32(WIDE_SCALE))
        assert len(o) == 1 and 200 < len(o[0]["points"]) < 500
        assert status[f] == 0 and n_kept[f] == 1 and src[f, 0] == 0
        assert np.array_equal(pts[f, off[f, 0]:off[f, 1]], o[0]["points"])
        assert np.abs(coef[f, 0] - o[0]["coef"]).max() < 2e-5
    for f in (2, 3):
        assert status[f] & 32, f


def test_voxel_key_range_through_compute_planes():
    """pslam_compute_planes_batch: a PEAC plane of ~1150 voxels 409.0 m deep (a 20000-pixel focal length, depth factor 100) matches the oracle; the same plane
    at 410 m lies beyond the 4095 depth keys and the call returns E_CAPACITY; so does a wall 33 m deep whose members reach x = -53 m under the 200-pixel
    focal length."""
    from planarslam_b200._lib import E_CAPACITY, PslamError
    from planarslam_b200.planes import ComputePlanes
    Kt, st = (20000.0, 20000.0, 319.5, 239.5), scale_of(100.0)
    deep = np.zeros((1, 480, 640), np.uint16)
    deep[0, 160:320, 240:400] = 40900
    res = ComputePlanes(_ctx(640, 480, 1, Kt, st), deep, 0.05, normals=False)
    assert _check_planes(res, deep, Kt, st) == 1 and 1000 < len(res[0]["points"][0]) < 2048
    deep[0, 160:320, 240:400] = 41000
    with pytest.raises(PslamError) as e:
        ComputePlanes(_ctx(640, 480, 1, Kt, st), deep, 0.05, normals=False)
    assert e.value.code == E_CAPACITY
    wide = np.zeros((1, 480, 640), np.uint16)
    wide[0, :, :120] = 33000
    with pytest.raises(PslamError) as e:
        ComputePlanes(_ctx(640, 480, 1, WIDE_K, WIDE_SCALE), wide, 0.05, normals=False)
    assert e.value.code == E_CAPACITY
