"""GPU: pslam_adapter::ref::FrameConstructor (include/pslam_reference_adapter.hpp) - the RGB-D Frame constructor as one call that fills the reference's own
Frame (src/Frame.cc, compiled into libmatch_ref.so) - against the reference's functions on the same inputs.

oracle/ref/frame_adapter_driver.cc (oracle/_ref/libframe_adapter_ref.so) turns arrays into cv::Mat inputs, runs the adapter and reads the Frame back; it
also runs the compiled ComputeImageBounds + AssignFeaturesToGrid, GetFeaturesInArea, ComputeStereoFromRGBD and isLineGood on reference Frames holding
the adapter's features.  ORB is compared with the compiled ORBextractor (liborb_ref.so).  The key lines, LBD rows, line functions, plane clouds,
coefficients and surface normals are compared with the records of pslam_frame_construct_batch, which the existing tests pin to cv2 4.13 LSD, the LBD
oracle and oracle/planepost.cc: PCL is absent, so that half is parity unpinned upstream."""
import ctypes as C
import os

import numpy as np
import pytest

import ref_lib
from cvtcolor_oracle import gray_from_color
from depth_cameras import CASES, frames, scale_of
from planarslam_b200._lib import KEYPOINT_DTYPE, Context
from planarslam_b200.frame import ConstructFrames, FrameOutputs
from planarslam_b200.lines import KEYLINE_DTYPE

LIB = os.path.join(ref_lib.REF_DIR, "libframe_adapter_ref.so")
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not (os.path.exists(os.path.join(ref_lib.REF_DIR, "libadapter_ref.so")) and os.path.exists(LIB)),
                                                  reason="oracle/_ref/libadapter_ref.so / libframe_adapter_ref.so not present")]
CAMS = [c for c, v in CASES.items() if v[:2] == (640, 480)] + ["odd_644x482", "min_120x117"]
BF, TH_DEPTH, PLANE_TH, CAP_PTS = 40.0, 40.0, 0.05, 16384
CV_16UC1, CV_32FC1, CV_8U, CV_32F = 2, 5, 0, 5
VOC = 0x5000                          # stored in mpORBvocabulary, never dereferenced
vp, i32, f32, f64, i64 = C.c_void_p, C.c_int, C.c_float, C.c_double, C.c_int64
_L = None


def lib():
    global _L
    if _L is None:
        ref_lib.match_lib()                       # the reference's Frame: the same instance (statics, libc rand) for both libraries
        L = C.CDLL(LIB)
        sig = {"fad_error": ([], C.c_char_p), "fad_create": ([i32, f32, i32, i32, i32, vp, vp, f32, f32, f32, f32, i32, i32, i32, i32, i32], vp),
               "fad_destroy": ([vp], None), "fad_frame": ([vp, vp, i32, vp, i32, f64, vp], vp), "fad_batch": ([vp, i32, vp, i32, vp, vp, vp, vp], i32),
               "fad_draws": ([vp], i64), "fad_advance": ([vp, i64], None), "fad_timing": ([vp, vp], None), "fad_extractor": ([vp], vp),
               "fad_free_frame": ([vp], None), "fad_extractor_tables": ([vp, vp], None), "fad_statics": ([vp], None), "fad_set_statics": ([i32, f32], None),
               "fad_scalars": ([vp, vp], None), "fad_sizes": ([vp, vp], None), "fad_scale_tables": ([vp, vp], None), "fad_keys": ([vp] * 6, None),
               "fad_grid": ([vp, vp, vp], None), "fad_features_in_area": ([vp, f32, f32, f32, i32, i32, vp], i32), "fad_lines": ([vp] * 6, None),
               "fad_vf3d": ([vp, vp, vp], i32), "fad_planes": ([vp] * 6, i32), "fad_normals": ([vp, vp], None), "fad_ref_grid_frame": ([vp, i32, i32], vp),
               "fad_ref_stereo": ([vp, vp, i32, i32, vp, vp], None), "fad_ref_is_line_good": ([vp, i32, vp, i32, i32, C.c_uint32, i64, vp, vp], None),
               "fad_rand_after": ([C.c_uint32, i64, vp], None), "fad_ref_track_local": ([vp, vp, vp, vp, f32, f32, vp, vp, vp, vp, vp], i32)}
        for name, (args, res) in sig.items():
            fn = getattr(L, name)
            fn.argtypes, fn.restype = args, res
        _L = L
    return _L


def statics():
    s = np.zeros(14)
    lib().fad_statics(s.ctypes.data)
    return s


class Adapter:
    def __init__(self, case, max_batch=1, rgb=True, dist=(0, 0, 0, 0), cap_plane_pts=CAP_PTS):
        w, h, K, factor, kw = CASES[case]
        self.w, self.h, self.K, self.scale = w, h, np.array(K, np.float32), scale_of(factor)
        self.nfeatures, self.nlevels = kw.get("nfeatures", 1000), kw.get("nlevels", 8)
        d = np.array(dist, np.float32)
        self.hnd = lib().fad_create(self.nfeatures, 1.2, self.nlevels, 20, 7, self.K.ctypes.data, d.ctypes.data, BF, TH_DEPTH, self.scale, PLANE_TH, w, h,
                                    int(rgb), max_batch, cap_plane_pts)
        if not self.hnd:
            raise ValueError(lib().fad_error().decode())

    def frame(self, image, depth, stamp, depth_type=CV_16UC1):
        im, d = np.ascontiguousarray(image, np.uint8), np.ascontiguousarray(depth)
        f = lib().fad_frame(self.hnd, im.ctypes.data, 1 if im.ndim == 2 else im.shape[2], d.ctypes.data, depth_type, stamp, VOC)
        if not f:
            raise ValueError(lib().fad_error().decode())
        return f

    def batch(self, images, depths, stamps):
        im, d, st = np.ascontiguousarray(images, np.uint8), np.ascontiguousarray(depths, np.uint16), np.ascontiguousarray(stamps, np.float64)
        out = (vp * len(im))()
        assert lib().fad_batch(self.hnd, len(im), im.ctypes.data, 1 if im.ndim == 3 else im.shape[3], d.ctypes.data, st.ctypes.data, VOC, out) == 0, \
            lib().fad_error().decode()
        return list(out)

    def draws(self):
        return lib().fad_draws(self.hnd)

    def close(self):
        lib().fad_destroy(self.hnd)


def read(f, w, h):
    """Every member FrameConstructor writes, as arrays."""
    L = lib()
    sc, sz = np.zeros(28), np.zeros(24, np.int64)
    L.fad_scalars(f, sc.ctypes.data)
    L.fad_sizes(f, sz.ctypes.data)
    n, nl, nlev, nku = int(sz[0]), max(int(sc[3]), 0), int(sz[21]), int(sz[1])
    r = {"scalars": sc, "sizes": sz}
    keys, keys_un, desc = np.zeros(n, KEYPOINT_DTYPE), np.zeros(nku, KEYPOINT_DTYPE), np.zeros((max(int(sz[4]), 0), 32), np.uint8)
    ur, dz = np.zeros(int(sz[2]), np.float32), np.zeros(int(sz[3]), np.float32)
    L.fad_keys(f, keys.ctypes.data, keys_un.ctypes.data, desc.ctypes.data, ur.ctypes.data, dz.ctypes.data)
    r.update(keys=keys, keys_un=keys_un, desc=desc, u_right=ur, depth=dz)
    tables = np.zeros((4, nlev), np.float32)
    L.fad_scale_tables(f, tables.ctypes.data)
    r["tables"] = tables
    off, idx = np.zeros(64 * 48 + 1, np.int32), np.zeros(max(n, 1), np.int32)
    L.fad_grid(f, off.ctypes.data, idx.ctypes.data)
    r["grid"] = (off, idx[:off[-1]])
    kl, lf, ld = np.zeros(nl, KEYLINE_DTYPE), np.zeros((nl, 3)), np.zeros((nl, 32), np.uint8)
    dl, l3 = np.zeros(nl, np.float32), np.zeros((nl, 6))
    L.fad_lines(f, kl.ctypes.data, lf.ctypes.data, ld.ctypes.data, dl.ctypes.data, l3.ctypes.data)
    r.update(keylines=kl, line_functions=lf, line_desc=ld, depth_line=dl, lines3d=l3)
    r["vf3d"] = vf3d(f)
    npts = L.fad_planes(f, None, None, None, None, None)
    npl = int(sz[17])
    poff, pts, wh, coef, meta = np.zeros(npl + 1, np.int32), np.zeros((npts, 3), np.float32), np.zeros((npl, 2), np.int32), np.zeros((npl, 4), np.float32), \
        np.zeros((npl, 3), np.int32)
    L.fad_planes(f, poff.ctypes.data, pts.ctypes.data, wh.ctypes.data, coef.ctypes.data, meta.ctypes.data)
    r.update(plane_off=poff, plane_pts=pts, plane_wh=wh, plane_coef=coef, plane_meta=meta)
    sn = np.zeros((int(sz[19]), 8), np.float32)
    L.fad_normals(f, sn.ctypes.data)
    r["normals"] = sn
    return r


def vf3d(f):
    L = lib()
    total = L.fad_vf3d(f, None, None)
    sz = np.zeros(24, np.int64)
    L.fad_sizes(f, sz.ctypes.data)
    head, pts = np.zeros((int(sz[20]), 15)), np.zeros((total, 27))
    L.fad_vf3d(f, head.ctypes.data, pts.ctypes.data)
    return head, pts


def same(a, b):
    """Identical members (NaN equal to NaN, bytes of structured records)."""
    assert a.keys() == b.keys()
    for k in a:
        x, y = a[k], b[k]
        if isinstance(x, tuple):
            for u, v in zip(x, y):
                assert np.array_equal(u, v, equal_nan=True), k
        elif x.dtype.names:
            assert x.tobytes() == y.tobytes(), k
        else:
            assert np.array_equal(x, y, equal_nan=True), k


def construct_records(case, gray, depth):
    w, h, K, factor, kw = CASES[case]
    ctx = Context(w, h, len(gray), fx=K[0], fy=K[1], cx=K[2], cy=K[3], depth_scale=scale_of(factor), **kw)
    return ConstructFrames(ctx, gray, depth, FrameOutputs(ctx, len(gray), cap_plane_pts=CAP_PTS), bf=BF, plane_dist_th=PLANE_TH, line_seed=1)


def sweep_queries(w, h, n=300, seed=0):
    rng = np.random.default_rng(seed)
    for _ in range(n):
        yield (float(rng.uniform(-20, w + 20)), float(rng.uniform(-20, h + 20)), float(rng.choice([3.0, 7.5, 15.0, 40.0, 100.0])),
               int(rng.integers(-1, 3)), int(rng.choice([-1, 0, 2, 7])))


def in_area(f, q):
    out = np.zeros(8192, np.int32)
    n = lib().fad_features_in_area(f, *q, out.ctypes.data)
    return out[:n].copy()


@pytest.mark.parametrize("case", CAMS)
def test_frame_constructor_members(case):
    w, h, K, factor, kw = CASES[case]
    L = lib()
    gray, depth = frames(case, 3)
    depth_m = (depth.astype(np.float32) * np.float32(scale_of(factor))).astype(np.float32)
    L.fad_set_statics(1, -99.0)
    A = Adapter(case)
    try:
        id0 = int(statics()[13])
        fs = [A.frame(gray[k], depth[k], 0.25 * k) for k in range(3)]
        draws = A.draws()
        recs = construct_records(case, gray, depth)
        ext_tables = np.zeros((4, A.nlevels), np.float32)
        L.fad_extractor_tables(A.hnd, ext_tables.ctypes.data)
        st = statics()
        fx, fy, cx, cy = (np.float32(v) for v in K)
        # statics: :73-78 and the first frame's :119-133
        assert np.array_equal(st[:6], [fx, fy, cx, cy, np.float32(1) / fx, np.float32(1) / fy])
        assert np.array_equal(st[6:12], [0, w, 0, h, np.float32(64) / np.float32(w), np.float32(48) / np.float32(h)]) and st[12] == 0
        refs, next4 = (vp * 3)(), np.zeros(4, np.int32)
        L.fad_ref_is_line_good((vp * 3)(*fs), 3, depth_m.ctypes.data, w, h, 1, 0, refs, next4.ctypes.data)
        adp4 = np.zeros(4, np.int32)
        L.fad_rand_after(1, draws, adp4.ctypes.data)
        assert np.array_equal(next4, adp4), "rand() position after three frames differs from three compiled isLineGood runs"
        n_valid = 0
        for k, f in enumerate(fs):
            r = read(f, w, h)
            sc, sz = r["scalars"], r["sizes"]
            n, nl, npl = int(sc[2]), int(sc[3]), int(sz[17])
            assert sc[0] == id0 + k and sc[1] == 0.25 * k and sc[4] == BF and sc[5] == np.float32(BF) / fx and sc[6] == TH_DEPTH
            assert sc[7] == A.nlevels and sc[8] == np.float32(1.2) and sc[9] == np.float32(np.log(np.float64(np.float32(1.2)))) and sc[10] == npl and sc[11] == 1
            assert np.array_equal(sc[12:21], [fx, 0, cx, 0, fy, cy, 0, 0, 1]) and np.array_equal(sc[21:25], [0, 0, 0, 0])
            assert sc[25] == VOC and sc[26] == L.fad_extractor(A.hnd) and sc[27] == 0
            assert np.array_equal(r["tables"], ext_tables), "scale tables differ from the extractor's getters"
            # 1. ORB against the compiled ORBextractor
            okps, odesc = ref_lib.ref_orb_extract(gray[k], A.nfeatures, 1.2, A.nlevels, 20, 7)
            assert n == len(okps) > 0 and r["keys"].tobytes() == okps.tobytes() and np.array_equal(r["desc"], odesc) and sz[23] == CV_8U
            assert r["keys_un"].tobytes() == r["keys"].tobytes()
            # 2. stereo against the compiled ComputeStereoFromRGBD on a Frame holding the adapter's key points
            ur, dz = np.zeros(n, np.float32), np.zeros(n, np.float32)
            L.fad_ref_stereo(f, depth_m[k].ctypes.data, w, h, ur.ctypes.data, dz.ctypes.data)
            assert np.array_equal(r["u_right"], ur) and np.array_equal(r["depth"], dz)
            # 3. image bounds, grid and GetFeaturesInArea against the compiled ComputeImageBounds + AssignFeaturesToGrid
            before = statics()
            R = L.fad_ref_grid_frame(f, w, h)
            try:
                assert np.array_equal(statics(), before)
                roff, ridx = np.zeros(64 * 48 + 1, np.int32), np.zeros(max(n, 1), np.int32)
                L.fad_grid(R, roff.ctypes.data, ridx.ctypes.data)
                assert np.array_equal(r["grid"][0], roff) and np.array_equal(r["grid"][1], ridx[:roff[-1]])
                hits = 0
                for q in sweep_queries(w, h, seed=k):
                    a, b = in_area(f, q), in_area(R, q)
                    assert np.array_equal(a, b), q
                    hits += len(a)
                assert hits > 100
            finally:
                L.fad_free_frame(R)
            # per-feature vectors (:113-116, :143-151)
            assert list(sz[:7]) == [n] * 7 and list(sz[7:9]) == [nl] * 2 and list(sz[9:17]) == [npl] * 8 and sz[18] == npl and sz[22] == 1
            # 4. isLineGood: the compiled function on the adapter's key lines, the three frames in a row from srand(1)
            rr = read(refs[k], w, h)
            assert np.array_equal(r["depth_line"], rr["depth_line"]) and np.array_equal(r["lines3d"], rr["lines3d"])
            for u, v in zip(r["vf3d"], rr["vf3d"]):
                assert np.array_equal(u, v), "mVF3DLines differ from the compiled isLineGood"
            n_valid += len(r["vf3d"][0])
            # 5. key lines, LBD rows, line functions, planes and normals against the frame-construct records
            assert nl == int(recs.n_lines[k]) > 0
            for name in KEYLINE_DTYPE.names:
                assert np.array_equal(r["keylines"][name], recs.keylines[k, :nl][name]), name
            assert np.array_equal(r["line_desc"], recs.line_desc[k, :nl]) and np.array_equal(r["line_functions"], recs.line_functions[k, :nl])
            if k == 0:      # the records start every frame at srand(1)
                assert np.array_equal(r["depth_line"], recs.lines3d[k, :nl]["depth"])
            assert npl == int(recs.n_planes[k])
            assert np.array_equal(r["plane_off"], recs.plane_pt_off[k, :npl + 1]) and np.array_equal(r["plane_pts"], recs.plane_pts[k, :recs.plane_pt_off[k, npl]])
            assert np.array_equal(r["plane_coef"], recs.plane_coef[k, :npl]) and (r["plane_meta"] == [CV_32F, 4, 1]).all()
            assert np.array_equal(r["plane_wh"][:, 0], np.diff(r["plane_off"])) and (r["plane_wh"][:, 1] == 1).all()
            assert np.array_equal(r["normals"], recs.surface_normals8[k], equal_nan=True)
        assert n_valid > 0
        for f in list(fs) + list(refs):
            L.fad_free_frame(f)
    finally:
        A.close()


def test_frame_constructor_batch_equals_per_frame_replay():
    """batch() over 2 x max_batch + 3 frames: every frame starts at the rand() position of the call's start; operator() rewound to that position
    before each frame must fill the same members.  mnId runs consecutively, draws() stays."""
    L = lib()
    mb = 3
    case = "tum3"
    w, h = CASES[case][:2]
    gray, depth = frames(case, 2 * mb + 3, zero_slot=4, seed=5)
    B, P = Adapter(case, max_batch=mb), Adapter(case)
    try:
        P.frame(gray[0], depth[0], 0.0)                 # moves P's stream away from 0
        L.fad_advance(B.hnd, 17)
        start = B.draws()
        id0 = int(statics()[13])
        fb = B.batch(gray, depth, 0.5 * np.arange(len(gray)))
        assert B.draws() == start
        for k, f in enumerate(fb):
            L.fad_advance(P.hnd, start - P.draws())
            g = P.frame(gray[k], depth[k], 0.5 * k)
            a, b = read(f, w, h), read(g, w, h)
            assert a["scalars"][0] == id0 + k
            a["scalars"][0] = b["scalars"][0] = 0
            a["scalars"][26] = b["scalars"][26] = 0       # each adapter holds its own extractor
            same(a, b)
            L.fad_free_frame(f)
            L.fad_free_frame(g)
    finally:
        B.close()
        P.close()


def test_frame_constructor_refusals_and_early_return():
    L = lib()
    case = "tum3"
    w, h = CASES[case][:2]
    gray, depth = frames(case, 1)
    with pytest.raises(ValueError, match="distort"):
        Adapter(case, dist=(0.2624, -0.9531, -0.0054, 0.0026))       # TUM fr1
    A = Adapter(case)
    try:
        n0 = statics()[13]
        with pytest.raises(ValueError, match="CV_16UC1"):
            A.frame(gray[0], depth[0].astype(np.float32), 0.0, depth_type=CV_32FC1)
        assert statics()[13] == n0
        # an all-flat grey frame: no key point, the early return of :106-107 (lines and planes ran; nothing after :106)
        L.fad_set_statics(1, -99.0)
        flat = np.full((h, w), 128, np.uint8)
        f = A.frame(flat, depth[0], 1.0)
        r = read(f, w, h)
        sc, sz = r["scalars"], r["sizes"]
        assert sc[2] == 0 and sc[10] == -12345 and sc[5] == np.float32(-1.5) and sc[11] == 1
        assert list(sz[:4]) == [0, 0, 0, 0] and sz[23] == -1 and list(sz[5:17]) == [0] * 12
        st = statics()
        assert st[0] == np.float32(CASES[case][2][0]) and st[12] == 1 and (st[6:12] == np.float32(-99.0)).all()
        recs = construct_records(case, flat[None], depth[:1])
        assert sz[17] == int(recs.n_planes[0]) > 0 and np.array_equal(r["normals"], recs.surface_normals8[0], equal_nan=True)
        L.fad_free_frame(f)
        # colour input: converted as GrabImageRGBD does, equal to the grey frame the cvtColor oracle gives
        rng = np.random.default_rng(3)
        for ch, rgb in ((3, True), (4, False)):
            col = np.clip(gray[0][..., None].astype(np.int16) + rng.integers(-40, 41, (h, w, ch)), 0, 255).astype(np.uint8)
            C_ = Adapter(case, rgb=rgb)
            try:
                a, b = C_.frame(col, depth[0], 2.0), A.frame(gray_from_color(col, rgb), depth[0], 2.0)
                ra, rb = read(a, w, h), read(b, w, h)
                assert ra["scalars"][2] > 0
                for k in ("keys", "desc", "keylines", "line_desc", "u_right"):
                    assert ra[k].tobytes() == rb[k].tobytes(), (ch, k)
                L.fad_free_frame(a)
                L.fad_free_frame(b)
            finally:
                C_.close()
    finally:
        A.close()
    # a capacity error names the frame and leaves no Frame behind
    T = Adapter(case, cap_plane_pts=2)
    try:
        n0 = statics()[13]
        with pytest.raises(ValueError, match=r"frame at 3\.5.*capacity"):
            T.frame(gray[0], depth[0], 3.5)
        assert statics()[13] == n0 and T.draws() == 0
    finally:
        T.close()


def test_adapted_frame_runs_the_reference_tracking_code():
    """The compiled ORBmatcher::SearchByProjection(F, points, th) (after SearchLocalPoints' frustum loop) and Optimizer::PoseOptimization(&F) on an adapted
    Frame return what they return on the Frame oracle/ref/match_driver.cc builds from the same arrays (key points, stereo fields, descriptors, statics, scale
    tables), against a map made from the frame's own key points with depth."""
    import oracle_lib
    from planarslam_b200 import synth_pose
    case = "tum3"
    w, h, K, _, _ = CASES[case]
    gray, depth = frames(case, 1, seed=7)
    L = lib()
    A = Adapter(case)
    try:
        f = A.frame(gray[0], depth[0], 0.0)
        r = read(f, w, h)
        keys, n = r["keys_un"], len(r["keys_un"])
        st = statics()
        fx, fy, cx, cy = (np.float32(v) for v in st[:4])
        # map: every second key point with depth, back-projected (Tcw = identity), descriptors with a few flipped bits
        rng = np.random.default_rng(11)
        sel = np.flatnonzero(r["depth"] > 0)[::2]
        z = r["depth"][sel].astype(np.float64)
        X = np.stack([(keys["x"][sel] - cx) * z / fx, (keys["y"][sel] - cy) * z / fy, z], 1).astype(np.float32)
        lvl = keys["octave"][sel].astype(np.float64)
        dist = np.linalg.norm(X.astype(np.float64), axis=1)
        desc = r["desc"][sel] ^ np.packbits(rng.random((len(sel), 256)) < 0.03, axis=1)
        m = dict(n=len(sel), pos=np.ascontiguousarray(X), normal=np.ascontiguousarray((X / dist[:, None]).astype(np.float32)),
                 max_distance=(dist * 1.2 ** lvl).astype(np.float32), min_distance=(dist * 1.2 ** lvl / 1.2 ** 7).astype(np.float32),
                 desc=np.ascontiguousarray(desc), skip=np.zeros(len(sel), np.uint8), has_obs=np.ones(len(sel), np.uint8))
        T = np.eye(4, dtype=np.float32)
        base = synth_pose.make_pose_problem(1, n_points=4, n_lines=0, n_planes=0, n_par=0, n_ver=0)
        T0 = np.eye(4, dtype=np.float32)
        T0[:3, 3] = (0.01, -0.02, 0.015)
        settings = np.array([base[k] for k in ("angle_info", "dist_info", "par_info", "ver_info", "plane_chi", "vp_chi")], np.float64)
        th, nnr = 3.0, 0.8
        # the adapted Frame
        am, ao, aT, an = np.full(n, -1, np.int32), np.zeros(n, np.uint8), np.zeros((4, 4), np.float32), C.c_int32()
        na = L.fad_ref_track_local(f, T.ctypes.data, T0.ctypes.data, C.byref(oracle_lib.map_points_struct(m)), th, nnr, settings.ctypes.data, am.ctypes.data,
                                   aT.ctypes.data, ao.ctypes.data, C.byref(an))
        # the Frame match_driver.cc builds from the same arrays
        fv = dict(n=n, keys_un=r["keys_un"], u_right=r["u_right"], desc=np.ascontiguousarray(r["desc"]), scale_factors=np.ascontiguousarray(r["tables"][0]),
                  Tcw=T, fx=float(fx), fy=float(fy), cx=float(cx), cy=float(cy), bf=BF, min_x=float(st[6]), max_x=float(st[7]), min_y=float(st[8]),
                  max_y=float(st[9]), log_scale_factor=float(r["scalars"][9]), n_levels=int(r["scalars"][7]))
        nr, rm, _ = ref_lib.ref_search_by_projection_map(fv, m, th, nnr, np.full(n, -1, np.int32))
        assert na == nr > 50 and np.array_equal(am, rm)
        idx = np.flatnonzero(rm >= 0)
        inv_s2 = r["tables"][3][keys["octave"][idx]]
        p = dict(base, Xw=np.ascontiguousarray(X[rm[idx]]), obs=np.ascontiguousarray(np.stack([keys["x"][idx], keys["y"][idx], r["u_right"][idx]], 1), np.float32),
                 inv_sigma2=np.ascontiguousarray(inv_s2, np.float32), fx=float(fx), fy=float(fy), cx=float(cx), cy=float(cy), bf=BF, Tcw0=T0)
        ro = ref_lib.ref_full_pose_optimization(p)
        assert an.value == ro["n_inliers"] > 0 and np.array_equal(aT, ro["Tcw"]) and np.array_equal(ao[idx], ro["outlier_pt"])
        L.fad_free_frame(f)
    finally:
        A.close()
