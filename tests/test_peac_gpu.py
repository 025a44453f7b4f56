"""GPU: PEAC plane extraction through the C ABI vs the CPU oracle — bit-exact labels, block statistics and planes."""
import numpy as np
import pytest

import oracle_lib
from planarslam_b200 import synth

pytestmark = pytest.mark.gpu
K = np.array([[535.4, 0, 320.1], [0, 539.2, 247.6], [0, 0, 1]], np.float32)
SCALE = np.float32(1.0 / 5000.0)


def _check_frame(res, depth, blocks=None, coarse=None, Kt=(535.4, 539.2, 320.1, 247.6), scale=SCALE):
    labels, planes, members = res
    orc = oracle_lib.PeacOracle(depth, Kt, scale)
    if blocks is not None:
        st, geo, n, valid = blocks
        assert np.array_equal(n, orc.blk_i[:, 0]) and np.array_equal(valid, orc.blk_i[:, 1])
        assert st.tobytes() == orc.blk_d[:, :9].copy().tobytes(), "block running sums differ"
        ok = n >= 4
        assert geo[ok].tobytes() == orc.blk_d[ok][:, 9:17].copy().tobytes(), "block PCA differs"
    if coarse is not None:
        bm, nc = coarse
        assert nc == orc.n_coarse and np.array_equal(bm, orc.coarse_blocks)
    assert len(planes) == len(orc.planes)
    assert np.array_equal(labels, orc.labels), "plane labels differ"
    for i, (d8, i2) in enumerate(orc.planes):
        assert planes["normal"][i].tobytes() == d8[0:3].tobytes() and planes["center"][i].tobytes() == d8[3:6].tobytes()
        assert planes["mse"][i] == d8[6] and planes["curvature"][i] == d8[7]
        assert planes["N"][i] == i2[0] and planes["rid"][i] == i2[1]
        assert np.array_equal(members[i], orc.membership[i])
    return len(planes)


def test_peac_matches_oracle_stage_by_stage():
    from planarslam_b200.planes import PlaneDetection
    pd = PlaneDetection(max_batch=4)
    depth = np.stack([synth.render_frame(2, f)[1] for f in (0, 17, 40, 55)])
    res = pd.run_batch(depth, K, SCALE)
    tot = 0
    for f in range(len(depth)):
        tot += _check_frame(res[f], depth[f], pd.debug_blocks(f), pd.debug_coarse(f))
    assert tot >= 8          # the room corner shows 2-3 planes per frame


def test_reference_call_shape():
    from planarslam_b200.planes import PlaneDetection
    pd = PlaneDetection()
    d = synth.render_frame(5, 3)[1]
    assert pd.readDepthImage(d, K, SCALE)
    pd.runPlaneDetection(480, 640)
    orc = oracle_lib.PeacOracle(d)
    assert pd.plane_num_ == len(orc.planes) >= 2
    assert np.array_equal(pd.membershipImg, orc.labels)
    assert not pd.readDepthImage(d.astype(np.float32), K, SCALE)      # wrong type -> False like :34-38


def test_peac_edge_cases():
    from planarslam_b200.planes import PlaneDetection
    pd = PlaneDetection(max_batch=3)
    rng = np.random.default_rng(3)
    empty = np.zeros((480, 640), np.uint16)                                   # no depth at all -> no planes
    flat = np.full((480, 640), 7000, np.uint16)                               # one fronto-parallel plane, exact ties in mse
    noisy = synth.render_frame(9, 1)[1].copy()
    noisy[rng.random(noisy.shape) < 0.01] = 0                                 # i.i.d. holes wipe most blocks
    depth = np.stack([empty, flat, noisy])
    res = pd.run_batch(depth, K, SCALE)
    assert len(res[0][1]) == 0 and (res[0][0] == -1).all()
    for f in range(3):
        _check_frame(res[f], depth[f], pd.debug_blocks(f), pd.debug_coarse(f))
    # ICL-NUIM intrinsics have fy < 0 (Examples/RGB-D/ICL.yaml:9): y flips sign, labels must still agree
    Ki = np.array([[481.2, 0, 319.5], [0, -480.0, 239.5], [0, 0, 1]], np.float32)
    pd2 = PlaneDetection()
    d = synth.render_frame(4, 2)[1]
    r = pd2.run_batch(d[None], Ki, SCALE)[0]
    _check_frame(r, d, Kt=(481.2, -480.0, 319.5, 239.5))
    # 1280x960 (config 5)
    pd3 = PlaneDetection()
    d = synth.render_frame(6, 2, width=1280, height=960)[1]
    K2 = K * 2
    K2[2, 2] = 1
    r = pd3.run_batch(d[None], K2, SCALE)[0]
    assert _check_frame(r, d, Kt=(1070.8, 1078.4, 640.2, 495.2)) >= 2
