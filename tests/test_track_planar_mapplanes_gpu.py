"""GPU: MapPlane::UpdateCoefficientsAndPoints inside the planar tracking chain (pslam_track_planar_set_map_plane_updates): after every frame, tracked or not,
each frame plane with a map plane association is merged into that map plane's cloud on the device, and the next frame's SearchMapByCoefficients reads the new
cloud (src/Tracking.cc:294-304, src/MapPlane.cc:335-366).

The map is the room corner's points and lines with ONLY THE FIRST KEY FRAME'S PLANES, so the clouds must grow as the camera moves.  Checks:
  - exact replay on the host from the chain's own outputs: starting from the uploaded clouds, for every frame t and frame plane i (ascending) with association
    j, cloud_j = oracle map_plane_update([(frame cloud i, T_t), (cloud_j, I)]); T_t = toSE3Quat(Tcw_out[t]).inverse() from the oracle's SE3Quat restatement
    (oracle/g2o_math.h through tests/host_harness/se3quat_inverse_host.cc), frame clouds from ConstructFrames.  Byte-identical to map_planes();
  - the reference chain of test_track_planar_gpu.py with the oracle update inserted after every frame: poses, mLastRcm and stats as close as that test asks,
    plane association rows equal on every frame;
  - two coplanar frame planes on one map plane (a zero-depth stripe splits the floor): merged one after the other;
  - capacity (a cloud close to the 4096-voxel limit, an oversized snapshot plane), mode off, persistence across calls and reset on re-upload."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_lib
import test_track_planar_gpu as tp
from planarslam_b200 import synth, synth_map, synth_pose
from planarslam_b200._lib import E_CAPACITY, Context, PslamError
from planarslam_b200.frame import ConstructFrames
from planarslam_b200.synth_planar_map import build_planar_map
from planarslam_b200.tracking import PLANAR_STATS, PlanarTracker, default_planar_params

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 64
MAX_PTS = 4096
I4 = np.eye(4)


@pytest.fixture(scope="module")
def se3inv(tmp_path_factory):
    out = tmp_path_factory.mktemp("se3quat") / "libse3quat_inverse_host.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-I", os.path.join(ROOT, "oracle"), "-o", str(out),
                    os.path.join(ROOT, "tests", "host_harness", "se3quat_inverse_host.cc")], check=True)
    L = C.CDLL(str(out))
    L.host_se3quat_inverse.argtypes = [C.c_void_p, C.c_void_p]
    L.host_se3quat_inverse.restype = None

    def f(T):
        T = np.ascontiguousarray(T, np.float32)
        o = np.zeros((4, 4), np.float64)
        L.host_se3quat_inverse(T.ctypes.data, o.ctypes.data)
        return o
    return f


@pytest.fixture(scope="module")
def setup():
    ctx = Context(640, 480, max_batch=N)
    frames = [synth.render_frame(2, f)[:2] for f in range(N)]
    m = build_planar_map(ctx, list(range(0, N, 8)))
    m["planes"] = build_planar_map(ctx, [0])["planes"]          # the first key frame's planes only
    gray, depth = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
    return ctx, gray, depth, m


def _frames(ctx, gray, depth):
    prm = default_planar_params()
    return ConstructFrames(ctx, gray, depth, depth_factor=prm.base.depth_factor, bf=prm.base.bf, plane_dist_th=prm.plane_dist_th, line_seed=prm.line_seed)


def _split(off, pts):
    return [pts[off[j]:off[j + 1]].copy() for j in range(len(off) - 1)]


def _frame_cloud(fr, t, i):
    return fr.plane_pts[t, fr.plane_pt_off[t, i]:fr.plane_pt_off[t, i + 1]]


def _replay(clouds, fr, poses, rows, se3inv, t0=0):
    """UpdateCoefficientsAndPoints after every frame on the host; a merge above MAX_PTS voxels leaves the cloud as it was.  Returns (clouds, overflows)."""
    clouds, over = list(clouds), []
    for t in range(len(poses)):
        T = se3inv(poses[t])
        npl = int(fr.n_planes[t0 + t])
        assert (rows[t, :, npl:] == -1).all(), t
        for i in range(npl):
            j = int(rows[t, 0, i])
            if j < 0:
                continue
            new = oracle_lib.map_plane_update([(_frame_cloud(fr, t0 + t, i), T), (clouds[j], I4)])
            if len(new) > MAX_PTS:
                over.append((t, j))
                continue
            clouds[j] = new
    return clouds, over


def _same(a, b):
    return len(a) == len(b) and all(x.shape == y.shape and np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(a, b))


def _upload(m):
    return _split(m["planes"]["pts_off"], m["planes"]["pts"])


def test_map_plane_updates_replay_exactly(setup, se3inv):
    ctx, gray, depth, m = setup
    tr = PlanarTracker(ctx, update_map_planes=True)
    tr.set_map(m)
    T0 = synth_map.true_pose(0).astype(np.float32)
    poses, Rcm, stats = tr.track(gray, depth, T0)
    rows = tr.plane_matches()
    assert rows.shape == (N, 3, ctx.L.pslam_peac_max_planes(ctx.h))
    got = _split(*tr.map_planes())
    want, over = _replay(_upload(m), _frames(ctx, gray, depth), poses, rows, se3inv)
    assert not over
    assert _same(got, want)
    sizes0 = [len(c) for c in _upload(m)]
    assert max(len(g) / s for g, s in zip(got, sizes0)) > 1.5, ([len(g) for g in got], sizes0)
    assert np.mean((rows[:, 0] >= 0).any(axis=1)) >= 0.75                    # most frames merge a plane
    for t in range(N):
        ea, et = synth_pose.pose_error(poses[t], synth_map.true_pose(t))
        assert ea < 5e-3 and et < 2e-2, (t, ea, et)
    print("map plane points: upload", sizes0, "after", N, "frames", [len(g) for g in got])


class _UpdatingRef(tp._Ref):
    """The reference functions of test_track_planar_gpu._reference_chain, with two steps of Track() that composition leaves out:
      - TrackLocalMap drops the parallel / vertical associations PoseOptimization flagged (src/Tracking.cc:2018-2030): done on the recorded rows after the
        local-map optimisation (`optimise`, translation_only False);
      - the map plane clouds SearchMapByCoefficients reads are updated after every frame by the oracle.  _reference_chain calls manhattan once at the start of
        each frame, and its SearchByProjection(cur, last) receives the last frame's final pose: the update of frame t (its associations are the merge of its
        plane_match calls) runs there.  plane_match refuses to run with an update pending and the test counts the updates, so a change of that composition's
        call order fails the test instead of moving or dropping updates."""
    fr, se3inv, planes0 = None, None, None

    def __init__(self):
        super().__init__()
        self.clouds, self.t, self.mp3, self.rows, self.pending = _upload(dict(planes=self.planes0)), -1, None, [], False
        self.n_updates, self.n_dropped = 0, 0

    def optimise(self, p, translation_only):
        r = super().optimise(p, translation_only)
        if not translation_only:
            for f, key in ((1, "outlier_par"), (2, "outlier_ver")):
                for k, i in enumerate(np.nonzero(self.mp3[f] >= 0)[0]):
                    if r[key][k]:
                        self.mp3[f, i] = -1
                        self.n_dropped += 1
        return r

    def manhattan(self, *a):
        if self.mp3 is not None:
            self.rows.append(self.mp3)
        self.t += 1
        npl = int(self.fr.n_planes[self.t])
        self.mp3, self.pending = np.full((3, npl), -1, np.int32), self.t > 0
        return super().manhattan(*a)

    def search_last(self, fv, lfr, *a):
        if self.pending:
            t, T = self.t - 1, self.se3inv(lfr["Tcw"])
            for i, j in enumerate(self.rows[t][0]):
                if j >= 0:
                    self.clouds[j] = oracle_lib.map_plane_update([(_frame_cloud(self.fr, t, i), T), (self.clouds[j], I4)])
            self.pending = False
            self.n_updates += 1
        return super().search_last(fv, lfr, *a)

    def plane_match(self, T, fc, P, prm):
        assert not self.pending, "frame %d matches planes before the previous frame's map plane update" % self.t
        off = np.zeros(len(self.clouds) + 1, np.int32)
        off[1:] = np.cumsum([len(c) for c in self.clouds])
        Pc = dict(P, pts_off=off, pts=np.ascontiguousarray(np.concatenate(self.clouds), np.float32))
        n, f3 = super().plane_match(T, fc, Pc, prm)
        self.mp3 = np.where(f3 >= 0, f3, self.mp3)
        return n, f3


def _with_tilted_plane(m):
    """m plus a map plane tilted 8 degrees from the floor, 1 m above it: the frames' floor planes associate with it as parallel (normals within 10 degrees,
    too far for a match); 8 degrees is far beyond the parallel edges' 0.1-degree sigma (Plane.ParallelInfo), so PoseOptimization flags them as outliers."""
    ax = np.array([1.0, 0.0, 1.0]) / np.sqrt(2.0)
    a = np.deg2rad(8.0)
    n0 = np.array([0.0, 1.0, 0.0])
    n = n0 * np.cos(a) + np.cross(ax, n0) * np.sin(a) + ax * np.dot(ax, n0) * (1 - np.cos(a))
    p0 = np.array([0.0, 0.2, 1.8])
    u = np.cross(n, ax); u /= np.linalg.norm(u)
    v = np.cross(n, u)
    g = np.stack(np.meshgrid(np.linspace(-1.5, 1.5, 24), np.linspace(-1.5, 1.5, 24)), -1).reshape(-1, 2)
    pts = (p0 + g[:, :1] * u + g[:, 1:] * v).astype(np.float32)
    coef = np.append(n, -n @ p0).astype(np.float32)
    if coef[3] < 0:
        coef = -coef
    P = m["planes"]
    planes = dict(coef=np.concatenate([P["coef"], coef[None]]), bad=np.append(P["bad"], np.uint8(0)), pts_off=np.append(P["pts_off"], P["pts_off"][-1] + len(pts)).astype(np.int32),
                  pts=np.concatenate([P["pts"], pts]))
    return dict(m, planes=planes)


@pytest.mark.parametrize("case", ["room", "tilted_plane"])
def test_map_plane_updates_match_the_reference_chain(setup, se3inv, monkeypatch, case):
    ctx, gray, depth, m = setup
    if case == "tilted_plane":
        m = _with_tilted_plane(m)
    prm = default_planar_params()
    fr = _frames(ctx, gray, depth)
    T0 = synth_map.true_pose(0).astype(np.float32)
    _UpdatingRef.fr, _UpdatingRef.se3inv, _UpdatingRef.planes0 = fr, staticmethod(se3inv), m["planes"]
    made = []
    monkeypatch.setattr(tp, "_Ref", lambda: made.append(_UpdatingRef()) or made[-1])
    ref = tp._reference_chain(fr, m, T0, prm)
    R = made[0]
    assert R.n_updates == N - 1 and len(R.rows) == N - 1
    ref_rows = R.rows + [R.mp3]
    print(case, "parallel / vertical associations dropped as outliers:", R.n_dropped)
    if case == "tilted_plane":
        assert R.n_dropped >= N // 4
    tr = PlanarTracker(ctx, prm, update_map_planes=True)
    tr.set_map(m)
    poses, Rcm, stats = tr.track(gray, depth, T0)
    rows = tr.plane_matches()
    worst = tp._compare(poses, Rcm, stats, ref)
    assert np.mean(np.all(stats == ref[2], axis=1)) >= 0.8, (stats[:6], ref[2][:6])
    for t in range(N):
        npl = int(fr.n_planes[t])
        assert np.array_equal(rows[t, :, :npl], ref_rows[t]) and (rows[t, :, npl:] == -1).all(), (t, rows[t, :, :npl], ref_rows[t])
    # the updated clouds take part: the device's clouds equal the replay of its own outputs, and they differ from the upload
    got = _split(*tr.map_planes())
    assert _same(got, _replay(_upload(m), fr, poses, rows, se3inv)[0]) and not _same(got, _upload(m))
    print("worst difference vs the reference chain with map plane updates (rad, m, mLastRcm):", worst)


def test_two_frame_planes_on_one_map_plane(setup, se3inv):
    ctx, gray, depth, m = setup
    n = 24
    g, d = gray[:n].copy(), depth[:n].copy()
    d[:, :, 420:444] = 0                 # a zero-depth stripe through the floor: PEAC returns the two halves as two coplanar planes
    tr = PlanarTracker(ctx, update_map_planes=True)
    tr.set_map(m)
    poses, _, _ = tr.track(g, d, synth_map.true_pose(0).astype(np.float32))
    rows = tr.plane_matches()
    fr = _frames(ctx, g, d)
    shared = [(t, j) for t in range(n) for j in set(rows[t, 0][rows[t, 0] >= 0].tolist()) if (rows[t, 0] == j).sum() >= 2]
    assert len(shared) >= n // 2, shared
    got = _split(*tr.map_planes())
    want, over = _replay(_upload(m), fr, poses, rows, se3inv)
    assert not over and _same(got, want)
    # not vacuous: merging both frame planes at once gives a different cloud than one after the other
    t, j = shared[0]
    before, _ = _replay(_upload(m), fr, poses[:t], rows[:t], se3inv)
    T = se3inv(poses[t])
    ii = [i for i in range(int(fr.n_planes[t])) if rows[t, 0, i] == j]
    joint = oracle_lib.map_plane_update([(_frame_cloud(fr, t, i), T) for i in ii] + [(before[j], I4)])
    seq = before[j]
    for i in ii:
        seq = oracle_lib.map_plane_update([(_frame_cloud(fr, t, i), T), (seq, I4)])
    assert not _same([joint], [seq])


def _track_raw(tr, gray, depth, T0):
    """pslam_track_planar_sequence without the error check: (return code, poses, Rcm, stats)."""
    ctx, n = tr.ctx, len(gray)
    g, d = np.ascontiguousarray(gray, np.uint8), np.ascontiguousarray(depth, np.uint16)
    T0 = np.ascontiguousarray(T0, np.float32)
    R0 = (T0[:3, :3].astype(np.float64) @ tr.R_cm.astype(np.float64)).astype(np.float32)
    poses, Rcm, stats = np.zeros((n, 4, 4), np.float32), np.zeros((n, 3, 3), np.float32), np.zeros((n, PLANAR_STATS), np.int32)
    rc = ctx.L.pslam_track_planar_sequence(ctx.h, g.ctypes.data, d.ctypes.data, n, C.byref(tr.params), T0.ctypes.data, None, R0.ctypes.data,
                                           poses.ctypes.data, Rcm.ctypes.data, stats.ctypes.data)
    return rc, poses, Rcm, stats


def _with_plane(m, j, cloud):
    clouds = _upload(m)
    clouds[j] = np.ascontiguousarray(cloud, np.float32).reshape(-1, 3)
    off = np.zeros(len(clouds) + 1, np.int32)
    off[1:] = np.cumsum([len(c) for c in clouds])
    return dict(m, planes=dict(m["planes"], pts_off=off, pts=np.concatenate(clouds)))


def test_capacity(setup, se3inv):
    ctx, gray, depth, m = setup
    n = 32
    T0 = synth_map.true_pose(0).astype(np.float32)
    # the floor plane (y = 1.2) a few voxels short of the limit: its cloud plus one point per voxel of a patch of the same plane far from the camera
    j = int(np.argmax(np.abs(m["planes"]["coef"][:, 1])))
    own = oracle_lib.map_plane_update([(_upload(m)[j], I4)])
    k = MAX_PTS - 2 - len(own)
    far = np.stack([20.05 + 0.1 * (np.arange(k) % 64), np.full(k, 1.2), 20.05 + 0.1 * (np.arange(k) // 64)], 1).astype(np.float32)
    near_full = oracle_lib.map_plane_update([(np.concatenate([_upload(m)[j], far]), I4)])
    assert len(near_full) == MAX_PTS - 2
    mc = _with_plane(m, j, near_full)
    tr = PlanarTracker(ctx, update_map_planes=True)
    tr.set_map(mc)
    rc, poses, Rcm, stats = _track_raw(tr, gray[:n], depth[:n], T0)
    assert rc == E_CAPACITY
    rows = tr.plane_matches(n)
    got = _split(*tr.map_planes())
    want, over = _replay(_upload(mc), _frames(ctx, gray[:n], depth[:n]), poses, rows, se3inv)
    assert over and all(jj == j for _, jj in over), over        # the merges that would overflow left the plane as it was
    assert _same(got, want) and len(got[j]) <= MAX_PTS
    # every output is written: the frames still track
    assert np.isfinite(poses).all() and np.isfinite(Rcm).all() and stats[:, 12].sum() > 0
    for t in range(n):
        ea, et = synth_pose.pose_error(poses[t], synth_map.true_pose(t))
        assert ea < 5e-3 and et < 2e-2, (t, ea, et)
    # a snapshot plane above the limit is refused in update mode, before any work; without updates it is accepted
    big = np.concatenate([near_full, far[:4] + np.float32([0, 0, -5.0])])
    assert len(big) > MAX_PTS
    tr.set_map(_with_plane(m, j, big))
    with pytest.raises(PslamError) as e:
        tr.track(gray[:2], depth[:2], T0)
    assert e.value.code == E_CAPACITY
    tr.update_map_planes = False
    tr.track(gray[:2], depth[:2], T0)


def test_mode_off_persistence_and_reset(setup, se3inv):
    ctx, gray, depth, m = setup
    T0 = synth_map.true_pose(0).astype(np.float32)
    plain = Context(640, 480, max_batch=N)
    tp0 = PlanarTracker(plain)
    tp0.set_map(m)
    p0, r0, s0 = tp0.track(gray, depth, T0)
    # switched on and off again: byte-identical to a context that never enabled updates, clouds = the upload
    tr = PlanarTracker(ctx, update_map_planes=True)
    assert PlanarTracker(ctx).update_map_planes and not PlanarTracker(plain).update_map_planes      # the setting belongs to the context
    tr.set_map(m)
    tr.track(gray[:4], depth[:4], T0)
    assert not _same(_split(*tr.map_planes()), _upload(m))
    tr.update_map_planes = False
    p1, r1, s1 = tr.track(gray, depth, T0)
    assert p0.tobytes() == p1.tobytes() and r0.tobytes() == r1.tobytes() and s0.tobytes() == s1.tobytes()
    assert _same(_split(*tr.map_planes()), _upload(m))
    # two calls continue from each other's clouds: the replay across both calls
    tr.update_map_planes = True
    h = N // 2
    pa, _, _ = tr.track(gray[:h], depth[:h], T0)
    ra = tr.plane_matches()
    pb, _, _ = tr.track(gray[h:], depth[h:], pa[-1])
    rb = tr.plane_matches()
    fr = _frames(ctx, gray, depth)
    mid, o1 = _replay(_upload(m), fr, pa, ra, se3inv)
    want, o2 = _replay(mid, fr, pb, rb, se3inv, t0=h)
    assert not o1 and not o2
    got = _split(*tr.map_planes())
    assert _same(got, want) and not _same(got, mid)
    # a re-upload resets the clouds
    tr.set_map(m)
    assert _same(_split(*tr.map_planes()), _upload(m))
    with pytest.raises(PslamError):
        PlanarTracker(plain).plane_matches(1)             # no call in update mode on this context


def test_matcher_reads_the_updated_clouds(setup):
    """SearchMapByCoefficients on the device reads the grown clouds, not the upload.  The floor map plane is uploaded with its cloud flattened 3.5 cm above
    the floor (a flat cloud: the minimum distance over noisy points would not show the offset): close enough for the frames' floor planes at the true pose.  A later frame whose pose is off by 3 cm in the other direction sees the floor 6.5 cm from
    the uploaded cloud (no match, the threshold is 5 cm) but ~3 cm from the floor points the earlier frames merged into it (a match)."""
    ctx, gray, depth, m = setup
    j = int(np.argmax(np.abs(m["planes"]["coef"][:, 1])))
    flat = _upload(m)[j].copy()
    flat[:, 1] = np.float32(1.2 - 0.035)                                         # world y points down: the floor is y = 1.2
    mo = _with_plane(m, j, flat)
    T0 = synth_map.true_pose(0).astype(np.float32)
    Td = T0.astype(np.float64)
    Td[:3, 3] -= Td[:3, :3] @ np.array([0.0, 0.03, 0.0])                        # camera centre 3 cm lower: the floor appears at y = 1.23
    Td = Td.astype(np.float32)
    tr = PlanarTracker(ctx, update_map_planes=True)
    tr.set_map(mo)
    tr.track(gray[:8], depth[:8], T0)
    assert (tr.plane_matches()[:, 0] == j).any(axis=1).all()                     # the floor was merged on every frame
    tr.track(gray[:1], depth[:1], Td)
    grown = tr.plane_matches()[0]
    tr.set_map(mo)                                                               # back to the uploaded clouds
    tr.track(gray[:1], depth[:1], Td)
    uploaded = tr.plane_matches()[0]
    assert (grown[0] == j).any() and not (uploaded[0] == j).any(), (grown, uploaded)
