"""GPU: the image half of the RGB-D Frame constructor - ORB (pyramid, blur, FAST, quadtree, descriptors), LSD with KeyLines and LBD, and PEAC (labels,
block statistics, planes, members) - at every camera and image size of depth_cameras.CASES, in batches, against the CPU oracle; and LSD on frames whose
rectangles are large enough that the NFA leaves both of its tables.

The sizes select kernel paths that the 640x480 tests never reach:
  * ORB blurs with the TMA kernel only when the width is a multiple of 16 and the frames are 16-byte aligned; 644x482 and 120x117 take k_blur_level, and
    at 644x482 a caller's odd frames start 8-byte aligned (the device-pointer call below passes such a frame).  At 640x480 and 1280x960 PSLAM_NO_TMA
    forces k_blur_level on the same frames, so the two blur kernels are compared with each other as well.
  * LSD scales by 0.8; at 640x481, 644x482 and 120x117 that is not a whole number of pixels (cvRound(0.8 * size), sampling step 1 / 0.8).
  * PEAC works on 10x10 blocks; 644x482, 640x481 and 120x117 end on partial blocks, whose pixels are labelled by the region growing alone.

Each case runs one batch of five frames (an odd count) with a flat gray frame and an all-zero depth frame in slot 2 and a real frame in the last slot of
max_batch, then a second call on the same context with three other frames, so state left from the first call would show: a sparse frame (few line
segments, few FAST corners), a piecewise-planar depth frame, and at the two smallest sizes a noise frame (more FAST candidates than the quota, so the
quadtree splits the largest nodes first).

Bar (as test_orb_gpu.py, test_lsd_gpu.py, test_lbd_gpu.py, test_peac_gpu.py): ORB key-point records and descriptors bit-exact, with every pyramid level,
blurred level and FAST candidate list; LSD segments, widths and precisions bit-exact and log-NFA to 1e-9; KeyLines exact except angle (3e-7); LBD floats
and descriptor bytes exact; PEAC labels, planes, members, block statistics and coarse maps bit-exact.  Where oracle/_ref holds the reference's own ORB
extractor and plane detector, the GPU results must equal theirs too."""

import numpy as np
import pytest

import oracle_lib
import ref_lib
from depth_cameras import CASES, frames, ramp_band, scale_of
from planarslam_b200 import synth
from test_peac_gpu import _check_frame

pytestmark = pytest.mark.gpu
f32 = np.float32
B, FLAT = 5, 2


def _sparse(w, h):
    g = np.full((h, w), 90, np.uint8)
    g[h // 5:h // 3, w // 3:w // 2] = 200
    g[3 * h // 5:2 * h // 3, w // 2:4 * w // 5] = 10
    return g


def _calls(case):
    """The two calls of a case, each (gray uint8 [n][h][w], depth uint16 [n][h][w]): B frames of the room sequence with a flat gray / all-zero depth frame in
    slot FLAT, then three frames of another sequence with the sparse gray frame and a piecewise-planar depth frame in slot 1, and at the two smallest sizes
    a noise gray frame in slot 2."""
    w, h, _, factor, _ = CASES[case]
    g1, d1 = frames(case, B, zero_slot=FLAT)
    g1[FLAT] = 128
    g2, d2 = frames(case, 3, seed=5)
    g2[1] = _sparse(w, h)
    pw = synth.piecewise_planar_depth(3, width=max(w, 200), height=max(h, 200), n_rect=6)[:h, :w]      # 1 / 5000 m units
    d2[1] = np.rint(pw * (factor / 5000.0)).astype(np.uint16)
    if w * h <= 320 * 240:
        g2[2] = np.random.default_rng(w).integers(0, 256, (h, w), dtype=np.uint8)
    return (g1, d1), (g2, d2)


def _orb_params(case):
    kw = CASES[case][4]
    return kw.get("nfeatures", 1000), kw.get("nlevels", 8)


def _check_orb_stages(ext, f, gray, nf, nl):
    orc = oracle_lib.OrbOracle(nf, 1.2, nl, 20, 7)
    orc.extract(gray)
    for l in range(nl):
        assert np.array_equal(ext.debug_level(f, l), orc.level(l)), (f, l)
        assert np.array_equal(ext.debug_level(f, l, blurred=True), oracle_lib.blur(orc.level(l))), (f, l)
        assert np.array_equal(ext.debug_candidates(f, l), orc.candidates(l)), (f, l)


@pytest.mark.parametrize("case", sorted(CASES))
def test_orb_matches_the_oracle(case, monkeypatch):
    from planarslam_b200.orb import ORBextractor
    w, h = CASES[case][:2]
    nf, nl = _orb_params(case)
    ext = ORBextractor(nf, 1.2, nl, 20, 7, max_batch=B)
    calls = _calls(case)
    first = None
    for call, (gray, _) in enumerate(calls):
        kps, desc = ext.extract_batch(gray)
        for f in range(len(gray)):
            ok, od = oracle_lib.orb_extract(gray[f], nf, 1.2, nl, 20, 7)
            assert len(kps[f]) == len(ok), (call, f, len(kps[f]), len(ok))
            assert kps[f].tobytes() == ok.tobytes() and np.array_equal(desc[f], od), (call, f)
            if call == 0 and f != FLAT:
                assert len(ok) > 0.4 * nf, (f, len(ok))
        if call == 0:
            assert len(kps[FLAT]) == 0
            for f in range(len(gray)):
                _check_orb_stages(ext, f, gray[f], nf, nl)
            first = (kps, desc)
        else:
            _check_orb_stages(ext, len(gray) - 1, gray[-1], nf, nl)
    gray = calls[0][0]
    if case in ("tum3", "config5"):
        # the per-level blur kernel on the frames the TMA kernel blurred above: the same bytes; then the TMA kernel again after both changes of frame count
        monkeypatch.setenv("PSLAM_NO_TMA", "1")
        kps, desc = ext.extract_batch(gray)
        for f in range(B):
            assert kps[f].tobytes() == first[0][f].tobytes() and np.array_equal(desc[f], first[1][f]), f
        _check_orb_stages(ext, B - 1, gray[B - 1], nf, nl)
        monkeypatch.delenv("PSLAM_NO_TMA")
        kps, desc = ext.extract_batch(gray)
        for f in range(B):
            assert kps[f].tobytes() == first[0][f].tobytes() and np.array_equal(desc[f], first[1][f]), f
    if case == "odd_644x482":
        # pslam_orb_extract_batch_dev from frame 1 of a device buffer: the base pointer is 8-byte aligned (644 * 482 = 8 mod 16)
        import torch
        dev = torch.device("cuda", 0)
        buf = torch.from_numpy(np.ascontiguousarray(gray[:2])).to(dev)
        base = buf.data_ptr() + w * h
        assert base % 16 == 8
        ctx = ext.context(h, w)
        cap = int(ctx.L.pslam_orb_max_keypoints(ctx.h))
        dk, dd = torch.zeros((cap, 28), dtype=torch.uint8, device=dev), torch.zeros((cap, 32), dtype=torch.uint8, device=dev)
        dn = torch.zeros(1, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        ctx.check(ctx.L.pslam_orb_extract_batch_dev(ctx.h, base, 1, dk.data_ptr(), dd.data_ptr(), cap, dn.data_ptr()))
        ctx.synchronize()
        n = int(dn.cpu()[0])
        assert n == len(first[0][1])
        assert dk[:n].cpu().numpy().tobytes() == first[0][1].tobytes() and np.array_equal(dd[:n].cpu().numpy(), first[1][1])


def _check_segments(res, gray, refine):
    for f in range(len(gray)):
        segs, width, prec, nfa = res[f]
        osegs, owidth, oprec, onfa = oracle_lib.lsd_detect(gray[f], refine, cap=65536)
        assert len(segs) == len(osegs), (refine, f, len(segs), len(osegs))
        assert np.array_equal(segs, osegs), (refine, f)
        assert np.array_equal(width, owidth) and np.array_equal(prec, oprec), (refine, f)
        assert np.allclose(nfa, onfa, rtol=1e-9, atol=1e-9), (refine, f)


@pytest.mark.parametrize("case", sorted(CASES))
def test_lsd_keylines_and_lbd_match_the_oracle(case):
    from planarslam_b200._lib import Context
    from planarslam_b200.lines import LineSegment
    w, h, _, _, kw = CASES[case]
    ls = LineSegment(ctx=Context(w, h, B, **kw))
    counts = []
    for call, (gray, _) in enumerate(_calls(case)):
        for refine in (0, 1, 2):
            _check_segments(ls.detect(gray, refine), gray, refine)
        if call == 0:
            for f in (1, B - 1):
                st, o = ls.debug_stage(f), oracle_lib.lsd_stages(gray[f], 2)
                assert st["scaled"].shape == (int(round(0.8 * h)), int(round(0.8 * w)))
                assert np.array_equal(st["scaled"], o["scaled"]), f
                assert np.array_equal(st["modgrad"][:-1, :-1], o["modgrad"][:-1, :-1]), f
                assert np.array_equal(st["angles"], o["angles"]), f
                defined = o["angles"].ravel()[o["order"]] != -1024.0
                assert np.array_equal(st["order"], o["order"][defined]), f
        kres = ls.ExtractLineSegment(gray, 40)
        lres = ls.ExtractLineSegmentWithDescriptors(gray, 40)
        for f in range(len(gray)):
            kl, lf = kres[f]
            okl, olf = oracle_lib.extract_line_segments(gray[f], 40)
            assert len(kl) == len(okl), (call, f, len(kl), len(okl))
            for name in kl.dtype.names:
                if name == "angle":
                    assert np.allclose(kl[name], okl[name], rtol=3e-7, atol=1e-7), (call, f)
                else:
                    assert np.array_equal(kl[name], okl[name]), (call, f, name)
            assert np.array_equal(lf, olf), (call, f)
            dkl, dlf, desc, lbd = lres[f]
            assert dkl.tobytes() == kl.tobytes() and np.array_equal(dlf, lf), (call, f)
            olbd, odesc = oracle_lib.lbd_compute(gray[f], kl)
            assert np.array_equal(lbd, olbd) and np.array_equal(desc, odesc), (call, f)
            counts.append(len(kl))
    assert counts[FLAT] == 0
    assert any(0 < n < 40 for n in counts), counts                   # a frame with fewer key lines than asked for


@pytest.mark.parametrize("case", sorted(CASES))
def test_peac_matches_the_oracle(case):
    from planarslam_b200.planes import PlaneDetection
    w, h, K, factor, kw = CASES[case]
    scale = f32(scale_of(factor))
    K33 = np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1]], f32)
    pd = PlaneDetection(max_batch=B, **({"nlevels": kw["nlevels"]} if "nlevels" in kw else {}))
    n_planes, partial = 0, 0
    for call, (_, depth) in enumerate(_calls(case)):
        res = pd.run_batch(depth, K33, scale)
        for f in range(len(depth)):
            n_planes += _check_frame(res[f], depth[f], pd.debug_blocks(f), pd.debug_coarse(f), Kt=K, scale=scale)
            labels = res[f][0]
            partial += int((labels[(h // 10) * 10:] >= 0).sum() + (labels[:, (w // 10) * 10:] >= 0).sum())
        if call == 0:
            assert len(res[FLAT][1]) == 0 and (res[FLAT][0] == -1).all()
    assert n_planes >= (1 if w * h < 320 * 240 else 2 * B)
    if h % 10 or w % 10:
        assert partial > 100, partial                                # pixels of the partial blocks were labelled and compared


def _ref_orb_and_peac(case):
    from planarslam_b200.orb import ORBextractor
    from planarslam_b200.planes import PlaneDetection
    _, _, K, factor, kw = CASES[case]
    nf, nl = _orb_params(case)
    scale = f32(scale_of(factor))
    ext = ORBextractor(nf, 1.2, nl, 20, 7, max_batch=B)
    pd = PlaneDetection(max_batch=B, **({"nlevels": kw["nlevels"]} if "nlevels" in kw else {}))
    K33 = np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1]], f32)
    for call, (gray, depth) in enumerate(_calls(case)):
        kps, desc = ext.extract_batch(gray)
        res = pd.run_batch(depth, K33, scale)
        for f in range(len(gray)):
            rk, rd = ref_lib.ref_orb_extract(gray[f], nf, 1.2, nl, 20, 7)          # src/ORBextractor.cc
            assert kps[f].tobytes() == rk.tobytes() and np.array_equal(desc[f], rd), (call, f)
            labels, planes, members = res[f]
            rl, rp, rm = ref_lib.ref_peac_run(depth[f], K, scale)                  # src/PlaneExtractor.cpp + include/peac/*.hpp
            assert np.array_equal(labels, rl) and len(planes) == len(rp), (call, f)
            for i, (d8, N) in enumerate(rp):
                assert planes["normal"][i].tobytes() == d8[0:3].tobytes() and planes["center"][i].tobytes() == d8[3:6].tobytes(), (call, f, i)
                assert planes["mse"][i] == d8[6] and planes["curvature"][i] == d8[7] and planes["N"][i] == N, (call, f, i)
                assert np.array_equal(members[i], rm[i]), (call, f, i)


@pytest.mark.skipif(ref_lib.orb_lib() is None or ref_lib.peac_lib() is None, reason="oracle/_ref/liborb_ref.so or libpeac_ref.so not present")
@pytest.mark.parametrize("case", sorted(CASES))
def test_orb_and_peac_identical_to_reference_code(case):
    _ref_orb_and_peac(case)


def _ramp_frames(w, h):
    return np.stack([ramp_band(w, h), ramp_band(w, h, 3.0), ramp_band(w, h, noise=8.0), ramp_band(w, h, 3.0, noise=8.0)])


@pytest.mark.parametrize("size", [(640, 480), (1280, 960)], ids=["640x480", "1280x960"])
def test_lsd_rectangles_beyond_the_nfa_tables(size):
    """One ramp band across the frame, axis-aligned (the dx == 0 branches of the rectangle code) and tilted by 3 degrees, clean and with noise: the NFA of
    rectangles of more than 8192 pixels comes from lsd_nfa_scalar's lsd_log_gamma1 branch (past the n <= 512 table and the n + 1 < 8192 log-gamma table)."""
    from planarslam_b200._lib import Context
    from planarslam_b200.lines import LineSegment
    w, h = size
    g = _ramp_frames(w, h)
    ls = LineSegment(ctx=Context(w, h, len(g)))
    for refine in (0, 1, 2):
        res = ls.detect(g, refine)
        _check_segments(res, g, refine)
        for f, (segs, width, _, _) in enumerate(res):
            assert 1 <= len(segs) <= 2, (refine, f, len(segs))
            length = np.hypot(segs[:, 2] - segs[:, 0], segs[:, 3] - segs[:, 1]).astype(np.float64)
            assert (length * width * 0.64).max() > 8192, (refine, f)        # rectangle pixels in the 0.8-scaled image
    segs = ls.detect(g[:1], 2)[0][0]
    assert len(segs) == 1 and segs[0, 0] == segs[0, 2]                     # the axis-aligned band gives an exactly vertical segment
