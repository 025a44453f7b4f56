"""GPU: the plane post-processing (pslam_planes_post_batch_dev: work list of the PEAC planes, persistent voxel / fit CTAs, compaction) on the shapes its
scheduling has to get right - bench-sized batches, frames without planes next to frames with many, planes rejected at each test, a plane above the 2048-voxel
capacity - against the CPU oracle (oracle/planepost.cc; bar as in test_planepost_gpu.py: same planes kept, voxel clouds exact, coefficients to 2e-5)."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib
from planarslam_b200 import synth

pytestmark = pytest.mark.gpu
K = synth.TUM3_K
SCALE = float(np.float32(1.0 / 5000.0))


def _ctx(n):
    from planarslam_b200._lib import Context
    return Context(640, 480, max_batch=n, fx=K[0], fy=K[1], cx=K[2], cy=K[3], depth_scale=SCALE)


def _check_against_oracle(depth, res):
    for f in range(len(depth)):
        o = oracle_lib.planes_post(depth[f])
        r = res[f]
        assert [p["src"] for p in o] == r["src"].tolist(), f
        for k, p in enumerate(o):
            assert np.array_equal(r["points"][k], p["points"]), (f, k)
            assert np.abs(r["coef"][k] - p["coef"]).max() < 2e-5, (f, k, r["coef"][k], p["coef"])


def _one_voxel_patch(d):
    d[250:398, 323:470] = int(0.35 * 5000)       # x, y in [0, 0.1) m, z = 0.35 m: PEAC finds a plane of ~22 k pixels whose cloud is one voxel
    return d


def test_sampled_sequence_frames_match_oracle():
    from planarslam_b200.planes import ComputePlanes
    frames = [0, 37, 90, 141, 199, 255]
    depth = np.stack([synth.render_frame(2, f, n_frames=256)[1] for f in frames])
    batch = np.concatenate([depth] * 4)                            # several records per plane index, frames repeated as in the benchmark's cycling
    res = ComputePlanes(_ctx(len(batch)), batch, 0.05, normals=False)
    for f in range(len(depth), len(batch)):
        a, b = res[f], res[f % len(depth)]
        assert a["src"].tolist() == b["src"].tolist() and np.array_equal(a["coef"], b["coef"])
        assert all(np.array_equal(p, q) for p, q in zip(a["points"], b["points"]))
    _check_against_oracle(depth, res[:len(depth)])
    assert sum(len(r["src"]) for r in res[:len(depth)]) >= 12


def test_frames_without_planes_between_frames_with_many():
    from planarslam_b200.planes import ComputePlanes
    empty = np.zeros((480, 640), np.uint16)
    depth = np.stack([empty, synth.piecewise_planar_depth(5, n_rect=11, curved=False), empty, empty, synth.render_frame(2, 17)[1], empty])
    res = ComputePlanes(_ctx(len(depth)), depth, 0.05, normals=False)
    for f in (0, 2, 3, 5):
        assert len(res[f]["src"]) == 0 and len(res[f]["coef"]) == 0
    assert len(res[1]["src"]) >= 5
    _check_against_oracle(depth, res)


def test_plane_of_fewer_than_three_voxels_is_dropped():
    from planarslam_b200.planes import ComputePlanes, PlaneDetection
    d = np.zeros((480, 640), np.uint16)
    d[20:200, 20:300] = 2 * 5000
    d = _one_voxel_patch(d)
    _, planes, _ = PlaneDetection().run_batch(d[None], np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1]], np.float32), np.float32(SCALE))[0]
    assert len(planes) == 2
    res = ComputePlanes(_ctx(1), d[None], 0.05, normals=False)
    assert res[0]["src"].tolist() == [0]
    _check_against_oracle(d[None], res)


def test_plane_above_voxel_capacity_sets_the_status_flag():
    from planarslam_b200._lib import E_CAPACITY, PslamError
    from planarslam_b200.planes import ComputePlanes
    wall = np.full((480, 640), 6 * 5000, np.uint16)            # a frontal wall at 6 m: ~3900 occupied voxels (oracle), above the 2048 slots
    assert len(oracle_lib.planes_post(wall)[0]["points"]) > 2048
    with pytest.raises(PslamError) as e:
        ComputePlanes(_ctx(2), np.stack([synth.render_frame(2, 5)[1], wall]), 0.05, normals=False)
    assert e.value.code == E_CAPACITY


def test_plane_beyond_the_distance_threshold_is_dropped():
    """The post-processing of device-resident PEAC results, once as PEAC left them and once with one plane record moved 0.3 m along its normal: that plane
    fails MaxPointDistanceFromPlane and disappears, everything else is unchanged."""
    import torch
    from planarslam_b200._lib import PLANE_DTYPE
    n, H, W = 3, 480, 640
    ctx = _ctx(n)
    L = ctx.L
    L.pslam_planes_post_batch_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 4 + [C.c_float] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
    maxp, cap = int(L.pslam_peac_max_planes(ctx.h)), 16384
    dev = torch.device("cuda", 0)
    depth = np.stack([synth.render_frame(2, f)[1] for f in (3, 40)] + [synth.piecewise_planar_depth(5, n_rect=11, curved=False)])
    d_depth = torch.from_numpy(depth.view(np.int16)).to(dev)
    d_labels, d_members = (torch.empty((n, H * W), dtype=torch.int32, device=dev) for _ in range(2))
    d_planes = torch.empty((n, maxp, PLANE_DTYPE.itemsize), dtype=torch.uint8, device=dev)
    d_npl, d_moff = torch.zeros(n, dtype=torch.int32, device=dev), torch.zeros((n, maxp + 1), dtype=torch.int32, device=dev)
    ctx.check(L.pslam_peac_run_batch_dev(ctx.h, d_depth.data_ptr(), n, d_labels.data_ptr(), d_planes.data_ptr(), d_npl.data_ptr(), d_members.data_ptr(),
                                         d_moff.data_ptr()))

    def post(planes):
        out = [torch.zeros(n, dtype=torch.int32, device=dev), torch.zeros((n, maxp), dtype=torch.int32, device=dev),
               torch.zeros((n, maxp, 4), dtype=torch.float32, device=dev), torch.zeros((n, maxp + 1), dtype=torch.int32, device=dev),
               torch.zeros((n, cap, 3), dtype=torch.float32, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)]
        ctx.check(L.pslam_planes_post_batch_dev(ctx.h, d_depth.data_ptr(), n, planes.data_ptr(), d_npl.data_ptr(), d_members.data_ptr(), d_moff.data_ptr(), 0.05,
                                                *[t.data_ptr() for t in out[:5]], cap, out[5].data_ptr()))
        ctx.synchronize()
        return [t.cpu().numpy() for t in out]

    ref = post(d_planes)
    f = 2
    assert ref[0][f] >= 2
    p = int(ref[1][f, 0])
    rec = d_planes.cpu().numpy().view(PLANE_DTYPE).reshape(n, maxp).copy()
    rec["center"][f, p] += 0.3 * rec["normal"][f, p]
    moved = post(torch.from_numpy(rec.view(np.uint8).reshape(n, maxp, -1)).to(dev))
    keep = [k for k in range(ref[0][f]) if ref[1][f, k] != p]
    assert moved[0][f] == len(keep) and moved[1][f, :len(keep)].tolist() == ref[1][f, keep].tolist()
    assert np.array_equal(moved[2][f, :len(keep)], ref[2][f, keep])
    for g in (0, 1):
        assert moved[0][g] == ref[0][g] and np.array_equal(moved[4][g], ref[4][g]) and np.array_equal(moved[2][g], ref[2][g])
    assert not moved[5].any() and not ref[5].any()
